"""CPU checks of the offline diarizer's prepare stage (no GPU needed):

* the oracle (``oracle/oracle_prepare.cpp``) against independent numpy / pure-Python restatements of the Swift sources:
  WeightInterpolation (with WeightInterpolationTests.swift case by case), the powerset decoder, processChunk;
* ``prepare_core.cuh`` — the arithmetic the kernels run — compiled for the host (``tests/emul/prepare_emul.cpp``) against
  the oracle, bit for bit;
* window arithmetic, argument validation and ``FA_STATUS_NO_DEVICE`` through the C ABI.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
FLT_MAX = np.finfo(np.float32).max


@pytest.fixture(scope="module")
def P():
    from oracle import oracle_prepare
    oracle_prepare.build()
    oracle_prepare.lib()
    return oracle_prepare


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("prepare") / "libprepare_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "prepare_emul.cpp")])
    L = C.CDLL(out)
    L.prepare_emul_decode.restype = C.c_longlong
    L.prepare_emul_decode.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.prepare_emul_resample.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
    L.prepare_emul_interp.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
    L.prepare_emul_speaker.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p] * 4
    L.prepare_emul_cosine.restype = C.c_float
    L.prepare_emul_cosine.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.prepare_emul_time.restype = C.c_double
    L.prepare_emul_time.argtypes = [C.c_double, C.c_int, C.c_double]
    return L


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---- independent restatements ---------------------------------------------------------------------------------------
def np_interp_table(n_in, n_out):
    """WeightInterpolation.swift:28-49 in numpy float32 (every array operation is one float32 rounding)."""
    scale = F32(n_out) / F32(n_in)
    pos = (np.arange(n_out, dtype=np.float32) + F32(0.5)) / scale - F32(0.5)
    clamped = np.minimum(np.maximum(pos, F32(0)), F32(n_in - 1))
    left = np.floor(clamped).astype(np.int32)
    right = np.minimum(left + 1, n_in - 1).astype(np.int32)
    w_right = clamped - left.astype(np.float32)
    return left, right, F32(1) - w_right, w_right


def np_resample(x, n_out):
    x = np.asarray(x, np.float32)
    if x.size == 0 or n_out <= 0:
        return np.zeros(0, np.float32)
    if x.size == n_out:
        return x.copy()
    l, r, wl, wr = np_interp_table(x.size, n_out)
    return x[l] * wl + x[r] * wr


def py_decode(logits, onset=0.5):
    """OfflineSegmentationProcessor.swift:321-405: argmax, weights, histogram exactly; log-probabilities in float64."""
    powerset = [[], [0], [1], [2], [0, 1], [0, 2], [1, 2], [0, 1, 2]]
    c, f, k = logits.shape
    best = np.zeros((c, f), np.int64)
    w = np.zeros((c, f, 3), np.float32)
    hist = np.zeros(8, np.int64)
    for ci in range(c):
        for fi in range(f):
            b, bv = 0, -FLT_MAX
            for cls in range(k):
                v = logits[ci, fi, cls]
                if v > bv:
                    bv, b = v, cls
            best[ci, fi] = b
            if b < 8:
                hist[b] += 1
            for s in powerset[min(b, 7)]:
                w[ci, fi, s] = 1.0
    x = logits.astype(np.float64)
    with np.errstate(all="ignore"):
        m = x.max(axis=2, keepdims=True)
        lse = np.log(np.exp(x - m).sum(axis=2, keepdims=True)) + m
        lp = x - lse
    return best, w, hist, lp, lse


def py_plan(w, offsets, frame_duration, total_samples, seg, plan):
    """OfflineEmbeddingExtractor.swift:421-707 in plain Python over float32 scalars."""
    chunks, frames, speakers = w.shape
    sr, win = seg["sample_rate"], seg["window_duration"]
    chunk_size = int(sr * win)
    thr = plan["skip_threshold"]
    skipping = thr >= 0
    entries, counters, cache, in_batch = [], dict(evaluated=0, empty=0, fallback=0, skipped=0), {}, 0
    branches = set()

    def fsum(v):
        s = F32(0)
        for x in v:
            s = F32(s + x)
        return s

    def cosine(a, b):
        dot, na, nb = fsum(a * b), fsum(a * a), fsum(b * b)
        den = F32(np.sqrt(na) * np.sqrt(nb))
        return F32(dot / den) if den > 0 else F32(0)

    for c in range(chunks):
        fd = frame_duration if frame_duration > 0 else win / max(1, frames)
        off = offsets[c] if c < len(offsets) and math.isfinite(offsets[c]) else c * win
        est = off * sr
        est = math.floor(abs(est) + 0.5) * (1 if est >= 0 else -1)
        start = max(0, min(int(est), total_samples))
        end = min(start + chunk_size, total_samples)
        if not start < end:
            branches.add("no_audio")
            continue
        min_frames = max(1, math.ceil(plan["min_segment_duration"] / fd)) if fd > 0 else 1
        cw = w[c]
        overlap = (cw > F32(1e-3)).sum(axis=1) > 1 if plan["exclude_overlap"] else np.zeros(frames, bool)
        for s in range(speakers):
            counters["evaluated"] += 1
            base = cw[:, s].copy()
            base_sum = fsum(base)
            if base_sum <= 0:
                counters["empty"] += 1
                branches.add("empty")
                continue
            clean = np.where(overlap, F32(0), base)
            clean_sum = fsum(clean)
            if clean_sum < F32(F32(frames) * F32(0.2)):
                counters["empty"] += 1
                branches.add("under_ratio")
                continue
            if clean_sum >= F32(min_frames):
                mask, mask_sum, fb = clean, clean_sum, 0
            else:
                mask, mask_sum, fb = base, base_sum, 1
                counters["fallback"] += 1
                branches.add("fallback")
            res = np_resample(mask, plan["weight_frames"])
            if fsum(res) <= 0:
                counters["empty"] += 1
                branches.add("zero_energy")
                continue
            reuse = -1
            if skipping and s in cache and cosine(mask, cache[s][1]) >= F32(thr):
                reuse = cache[s][0]
                counters["skipped"] += 1
                branches.add("reuse_hit")
            elif skipping:
                branches.add("reuse_miss" if s in cache else "reuse_first")
                cache[s] = (len(entries), mask)
            act = np.flatnonzero(mask > F32(1e-3))
            first = int(act[0]) if act.size else 0
            last = int(act[-1]) if act.size else first
            entries.append(dict(chunk=c, speaker=s, first=first, last=last, start=off + first * fd,
                                end=off + (last + 1) * fd, mask_sum=mask_sum, fallback=fb, reuse=reuse, mask=mask, res=res))
        in_batch += 1
        if in_batch == plan["fbank_batch"]:
            in_batch = 0
            if cache:
                branches.add("cache_cleared")
            cache.clear()
    return entries, counters, branches


def assert_plan_equal(got, entries, counters):
    assert got.count == len(entries)
    for name, key in (("chunk_index", "chunk"), ("speaker_index", "speaker"), ("start_frame", "first"),
                      ("end_frame", "last"), ("used_fallback", "fallback"), ("reuse_of", "reuse")):
        assert getattr(got, name).tolist() == [e[key] for e in entries], name
    assert got.start_time.tolist() == [e["start"] for e in entries]
    assert got.end_time.tolist() == [e["end"] for e in entries]
    assert np.array_equal(bits(got.mask_sum), bits([e["mask_sum"] for e in entries]))
    if entries:
        assert np.array_equal(bits(got.frame_weights), bits(np.stack([e["mask"] for e in entries])))
        assert np.array_equal(bits(got.model_weights), bits(np.stack([e["res"] for e in entries])))
    assert got.counters.tolist() == [counters[k] for k in ("evaluated", "empty", "fallback", "skipped")]


# ---- fixtures in data -------------------------------------------------------------------------------------------------
def branch_weights(frames=100, chunks=12):
    """Binary weights whose chunks enter every branch of processChunk (3 local speakers)."""
    w = np.zeros((chunks, frames, 3), np.float32)
    q = frames // 10
    w[0, :6 * q, 0] = 1                                    # speaker 0 alone; speakers 1, 2 empty
    w[1, :5 * q, 0] = 1; w[1, q:5 * q, 1] = 1              # 1 only inside the overlap: clean under 20 %
    w[2, :4 * q, 0] = 1; w[2, 3 * q:7 * q, 1] = 1          # both keep 30 % clean: fallback when min_frames is larger
    w[3, :3 * q, 0] = 1                                    # active only at the start: zero energy at weight_frames 1
    for k in range(4, chunks):                             # a mask that grows by 4 % per chunk: the reuse drift
        w[k, :int(frames * (0.4 + 0.04 * (k - 4))), 2] = 1
    return w


GRID = [(4, 4), (2, 4), (4, 2), (16, 7), (7, 16), (5, 1), (1, 5), (1, 1), (589, 998), (998, 589), (589, 589), (589, 1499),
        (589, 1), (3, 1000), (1000, 3), (31, 33), (33, 31)]


# ---- 1. interpolation ---------------------------------------------------------------------------------------------------
def test_interpolation_table_equals_numpy_restatement(P):
    for n_in, n_out in GRID:
        got, ref = P.interp_table(n_in, n_out), np_interp_table(n_in, n_out)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), (n_in, n_out)
        assert np.array_equal(bits(got[2]), bits(ref[2])) and np.array_equal(bits(got[3]), bits(ref[3])), (n_in, n_out)
        x = np.random.default_rng(n_in * 7 + n_out).uniform(0, 1, (3, n_in)).astype(np.float32)
        assert np.array_equal(bits(P.weight_resample(x, n_out)), bits(np.stack([np_resample(r, n_out) for r in x])))


def test_weight_interpolation_swift_cases(P):
    """WeightInterpolationTests.swift, case by case, on the oracle."""
    r = lambda x, n: P.weight_resample(np.asarray(x, np.float32), n)
    assert r([1, 2, 3, 4], 4).tolist() == [1, 2, 3, 4]                                  # identity
    up = r([0, 1], 4)
    assert up.size == 4 and up[0] < up[3] and (up >= 0).all() and (up <= 1).all()       # upsampling
    down = r([0, 0.5, 1, 0.5], 2)
    assert down.size == 2 and (down >= 0).all() and (down <= 1).all()                   # downsampling
    assert np.allclose(r([0, 10, 20, 30], 2), [5, 25], atol=1e-5)                       # half-pixel mapping
    x = np.arange(16, dtype=np.float32) * 0.25
    l, rr, wl, wr = P.interp_table(16, 7)
    assert np.allclose(r(x, 7), x[l] * wl + x[rr] * wr, atol=1e-5)                      # coefficients
    two = r([[1, 2, 3], [4, 5, 6]], 5)
    assert np.allclose(two[0], r([1, 2, 3], 5), atol=1e-6) and np.allclose(two[1], r([4, 5, 6], 5), atol=1e-6)
    assert np.allclose(r([[1, 3, 5, 7], [2, 4, 6, 8]], 2), [[2, 6], [3, 7]], atol=1e-5)  # broadcast rows


def test_python_mirror_guards_need_no_device(lib):
    """The empty cases of WeightInterpolationTests.swift and the zoom lengths are decided before any device work."""
    from fluidaudio_b200.segmentation import WeightInterpolation as W
    assert W.resample([], 5).size == 0 and W.resample([1, 2, 3], 0).size == 0
    assert W.resample_2d([], 5).size == 0
    assert W.zoom([], 2.0).size == 0 and W.zoom([1, 2, 3], 0).size == 0


# ---- 2. decode ----------------------------------------------------------------------------------------------------------
def decode_inputs(classes, rng):
    x = rng.standard_normal((4, 40, classes)).astype(np.float32) * 4
    x[1, :10] = np.round(x[1, :10])                       # ties
    x[1, 10:20] = 1.5
    x[2, 0] = -np.inf
    x[2, 1, 0] = np.inf
    x[2, 2, classes - 1] = np.inf
    x[2, 3] = np.nan
    x[2, 4, 0] = np.nan
    x[2, 5, classes // 2] = np.nan
    x[2, 6] = -FLT_MAX
    return x


@pytest.mark.parametrize("classes", [1, 7, 8, 11])
def test_oracle_decode_equals_restatement(P, classes):
    x = decode_inputs(classes, np.random.default_rng(classes))
    got = P.seg_decode(x)
    best, w, hist, lp, lse = py_decode(x)
    assert np.array_equal(got.speaker_weights, w) and np.array_equal(got.class_histogram, hist)
    assert hist.sum() == (best < 8).sum()
    ok = np.isfinite(lp) & np.isfinite(lse)
    bar = 2 * 2.0 ** -23 * (np.abs(lse) + np.abs(x.astype(np.float64)) + 1)   # 2 ulp of |lse| + |logit| (+ 1)
    assert ok.sum() > 0.9 * ok.size * (1 if classes > 1 else 0.5)
    assert (np.abs(got.log_probs.astype(np.float64) - lp)[ok] <= np.broadcast_to(bar, lp.shape)[ok]).all()
    sp = np.clip(1 - np.exp(got.log_probs[..., 0].astype(np.float64)), 0, 1)
    sure = np.isfinite(sp) & (np.abs(sp - 0.5) > 1e-5)
    assert np.array_equal((got.speech_probability >= 0.5)[sure], (sp >= 0.5)[sure])
    assert got.speech_frames == int((got.speech_probability >= 0.5).sum())


# ---- 3. plan ------------------------------------------------------------------------------------------------------------
PLAN_CASES = [
    dict(plan=dict(weight_frames=151), fd=0.1),
    dict(plan=dict(weight_frames=151, exclude_overlap=False), fd=0.1),
    dict(plan=dict(weight_frames=100, min_segment_duration=3.5), fd=0.1),                  # fallback
    dict(plan=dict(weight_frames=1), fd=0.1),                                               # zero energy
    dict(plan=dict(weight_frames=151, skip_threshold=0.95), fd=0.1),                        # reuse, pinned
    dict(plan=dict(weight_frames=151, skip_threshold=0.95, fbank_batch=3), fd=0.1),         # cache cleared
    dict(plan=dict(weight_frames=151, skip_threshold=1.0), fd=0.0),
    dict(plan=dict(weight_frames=151, skip_threshold=0.0), fd=0.1, total=16000 * 15),       # chunks without audio
    dict(plan=dict(weight_frames=151), fd=0.1, offsets=[0.0, math.nan, 4.0, math.inf]),     # non-finite, missing
]


def test_oracle_plan_equals_restatement_on_every_branch(P):
    seg = dict(P.SEG_DEFAULTS)
    w = branch_weights()
    seen = set()
    for case in PLAN_CASES:
        plan = {**P.PLAN_DEFAULTS, **case["plan"]}
        offsets = np.asarray(case.get("offsets", np.arange(w.shape[0]) * 2.0), np.float64)
        total = case.get("total", 16000 * 60)
        got = P.embedding_plan(w, offsets, case["fd"], total, seg, plan)
        entries, counters, branches = py_plan(w, offsets, case["fd"], total, seg, plan)
        assert_plan_equal(got, entries, counters)
        seen |= branches
    assert seen >= {"no_audio", "empty", "under_ratio", "fallback", "zero_energy", "reuse_hit", "reuse_miss",
                    "reuse_first", "cache_cleared"}, seen
    # pinned to the generating mask: the growing mask of chunks 4.. reuses chunk 4's entry until it has drifted, then
    # starts again from the chunk that missed -- a rolling comparison would never miss
    got = P.embedding_plan(w, np.arange(12) * 2.0, 0.1, 16000 * 60, seg, {**P.PLAN_DEFAULTS, "weight_frames": 151,
                                                                           "skip_threshold": 0.95})
    mine = got.speaker_index == 2
    gens = np.flatnonzero(mine & (got.reuse_of < 0))
    assert gens.size >= 2 and set(got.reuse_of[mine & (got.reuse_of >= 0)].tolist()) <= set(gens.tolist())


def test_oracle_plan_random_binary_weights(P):
    rng = np.random.default_rng(9)
    seg = dict(P.SEG_DEFAULTS)
    for frames, speakers, wf in ((1, 1, 1), (5, 3, 7), (50, 4, 50), (64, 3, 90)):
        w = (rng.random((9, frames, speakers)) < rng.random((9, 1, speakers))).astype(np.float32)
        for thr in (-1.0, 0.9):
            plan = {**P.PLAN_DEFAULTS, "weight_frames": wf, "skip_threshold": thr, "fbank_batch": 4,
                    "min_segment_duration": 0.5}
            got = P.embedding_plan(w, np.arange(9) * 2.0, 0.0, 16000 * 30, seg, plan)
            assert_plan_equal(got, *py_plan(w, np.arange(9) * 2.0, 0.0, 16000 * 30, seg, plan)[:2])


# ---- 4. the kernels' arithmetic on the host -----------------------------------------------------------------------------
def test_kernel_arithmetic_equals_oracle(P, emul):
    for n_in, n_out in GRID:
        ref = P.interp_table(n_in, n_out)
        got = (np.zeros(n_out, np.int32), np.zeros(n_out, np.int32), np.zeros(n_out, np.float32), np.zeros(n_out, np.float32))
        emul.prepare_emul_interp(n_in, n_out, *[g.ctypes.data for g in got])
        assert all(np.array_equal(g.view(np.uint32), r.view(np.uint32)) for g, r in zip(got, ref)), (n_in, n_out)
        x = np.random.default_rng(n_in + n_out).uniform(0, 1, (2, n_in)).astype(np.float32)
        out = np.zeros((2, n_out), np.float32)
        emul.prepare_emul_resample(x.ctypes.data, 2, n_in, n_out, out.ctypes.data)
        assert np.array_equal(bits(out), bits(P.weight_resample(x, n_out)))
    for classes in (1, 7, 8, 11):
        x = decode_inputs(classes, np.random.default_rng(classes + 20))
        ref = P.seg_decode(x)
        lp, w, hist = np.zeros_like(x), np.zeros(x.shape[:2] + (3,), np.float32), np.zeros(8, np.int64)
        speech = emul.prepare_emul_decode(x.ctypes.data, x.shape[0] * x.shape[1], classes, 0.5, lp.ctypes.data,
                                          w.ctypes.data, hist.ctypes.data)
        assert np.array_equal(w, ref.speaker_weights) and np.array_equal(hist, ref.class_histogram)
        assert np.array_equal(bits(lp), bits(ref.log_probs)) and speech == ref.speech_frames   # same libm on the host
    assert emul.prepare_emul_time(12.3, 77, 10.0 / 589) == 12.3 + 77.0 * (10.0 / 589)


def test_kernel_mask_decisions_equal_oracle(P, emul):
    seg = dict(P.SEG_DEFAULTS)
    w = branch_weights()
    chunks, frames, speakers = w.shape
    for case in PLAN_CASES[:4]:
        plan = {**P.PLAN_DEFAULTS, **case["plan"]}
        ref = P.embedding_plan(w, np.arange(chunks) * 2.0, case["fd"], 16000 * 60, seg, plan)
        min_frames = max(1, math.ceil(plan["min_segment_duration"] / case["fd"]))
        wf, n, fallbacks = plan["weight_frames"], 0, 0
        for c in range(chunks):
            for s in range(speakers):
                mask, res, out, sums = np.zeros(frames, np.float32), np.zeros(wf, np.float32), np.zeros(5, np.int32), \
                    np.zeros(3, np.float32)
                emul.prepare_emul_speaker(w[c].ctypes.data, frames, speakers, s, int(plan["exclude_overlap"]), min_frames, wf,
                                          mask.ctypes.data, res.ctypes.data, out.ctypes.data, sums.ctypes.data)
                fallbacks += out[1]
                if not out[0]:
                    continue
                assert (ref.chunk_index[n], ref.speaker_index[n], ref.start_frame[n], ref.end_frame[n],
                        ref.used_fallback[n]) == (c, s, out[2], out[3], out[1])
                assert np.array_equal(bits(mask), bits(ref.frame_weights[n])) and np.array_equal(bits(res), bits(ref.model_weights[n]))
                assert bits(sums[:1])[0] == bits(ref.mask_sum[n:n + 1])[0]
                n += 1
        assert n == ref.count and fallbacks == ref.counters[2]
    rng = np.random.default_rng(4)
    for _ in range(20):                                     # binary masks: the cosine is exact in any order
        a, b = (rng.random(589) < 0.4).astype(np.float32), (rng.random(589) < 0.6).astype(np.float32)
        dot, na, nb = F32((a * b).sum()), F32(a.sum()), F32(b.sum())
        want = F32(dot / F32(np.sqrt(na) * np.sqrt(nb)))
        assert emul.prepare_emul_cosine(a.ctypes.data, b.ctypes.data, 589) == want


# ---- 5. windows ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [dict(), dict(step_ratio=0.1), dict(sample_rate=8000, window_duration=5.0, step_ratio=0.33),
                                 dict(window_duration=0.001, step_ratio=0.01)])
def test_window_counts_and_offsets(P, lib, cfg):
    from fluidaudio_b200.segmentation import OfflineSegmentationProcessor, SegmentationConfig
    proc = OfflineSegmentationProcessor(SegmentationConfig(**cfg))
    _, window, step = proc.window_count(1)
    assert window == int(proc.config.sample_rate * proc.config.window_duration)
    assert step == max(1, int(window * proc.config.step_ratio))
    for total in (0, 1, window - 1, window, window + 1, 3 * step + 7, 10 * window + step // 2):
        if total < 0:
            continue
        assert proc.window_count(total) == P.seg_window_count(total, **{**P.SEG_DEFAULTS, **cfg})
        assert proc.window_count(total)[0] == len(range(0, total, step))
    audio = synth.tone_noise_audio(2 * window + 3)
    wins, offs = P.seg_windows(audio, **{**P.SEG_DEFAULTS, **cfg})
    assert offs.tolist() == [o / proc.config.sample_rate for o in range(0, audio.size, step)]
    for i, o in enumerate(range(0, audio.size, step)):
        seg = audio[o:o + window]
        assert np.array_equal(wins[i, :seg.size], seg) and not wins[i, seg.size:].any()


# ---- 6. the C ABI before any device work --------------------------------------------------------------------------------
def test_argument_validation_needs_no_device(lib):
    seg, plan = _lib.SegConfig(), _lib.EmbedPlanConfig()
    lib.fa_seg_default_config(C.byref(seg))
    lib.fa_embed_plan_default_config(C.byref(plan))
    assert (seg.sample_rate, seg.window_duration, seg.step_ratio, seg.speech_onset_threshold) == (16000, 10.0, 0.2, 0.5)
    assert (plan.exclude_overlap, plan.min_segment_duration, plan.weight_frames, plan.audio_sample_count,
            plan.fbank_batch) == (1, 1.0, 589, 160000, 32) and plan.skip_threshold < 0
    n, one = C.c_int32(7), np.zeros(8, np.float32)
    p = one.ctypes.data
    assert lib.fa_seg_window_count(-1, C.byref(seg), C.byref(n), None, None) == 1
    assert lib.fa_seg_window_count(5, None, C.byref(n), None, None) == 1
    for field, bad in (("step_ratio", 0.0), ("step_ratio", 1.5), ("window_duration", 0.0), ("sample_rate", 0)):
        broken = _lib.SegConfig()
        lib.fa_seg_default_config(C.byref(broken))
        setattr(broken, field, bad)
        assert lib.fa_seg_window_count(5, C.byref(broken), C.byref(n), None, None) == 1, field
        assert lib.fa_seg_decode(p, 1, 1, 7, C.byref(broken), None, p, None, None) == 1
    assert lib.fa_seg_windows(p, 0, C.byref(seg), 0, 0, p, None) == 5                   # noSpeechDetected
    assert b"noSpeechDetected" in lib.fa_last_error()
    assert lib.fa_seg_windows(p, 8, C.byref(seg), 0, 2, p, None) == 1                   # past the last window
    assert lib.fa_seg_windows(p, 8, C.byref(seg), 0, 0, p, None) == 0
    assert lib.fa_seg_windows(None, 8, C.byref(seg), 0, 1, p, None) == 1
    for classes in (0, 17):
        assert lib.fa_seg_decode(p, 1, 1, classes, C.byref(seg), None, p, None, None) == 1
    hist, speech = np.ones(8, np.int64), C.c_int64(3)
    assert lib.fa_seg_decode(None, 0, 5, 7, C.byref(seg), None, None, hist.ctypes.data, C.byref(speech)) == 0
    assert not hist.any() and speech.value == 0
    assert lib.fa_seg_decode(None, 1, 1, 7, C.byref(seg), None, p, None, None) == 1
    plan_args = lambda w, c, f, s, cfg, cnt: lib.fa_embedding_plan(w, c, f, s, None, 0, 0.0, 100, C.byref(seg), cfg,
                                                                   *([None] * 11), cnt, None)
    assert plan_args(p, 1, 1, 1, C.byref(plan), None) == 1
    assert plan_args(None, 0, 5, 3, C.byref(plan), C.byref(n)) == 0 and n.value == 0    # empty input: zero entries
    assert plan_args(p, 3, 0, 3, C.byref(plan), C.byref(n)) == 0 and n.value == 0
    assert plan_args(None, 1, 1, 1, C.byref(plan), C.byref(n)) == 1
    assert plan_args(p, -1, 1, 1, C.byref(plan), C.byref(n)) == 1
    for field in ("weight_frames", "audio_sample_count", "fbank_batch"):
        broken = _lib.EmbedPlanConfig()
        lib.fa_embed_plan_default_config(C.byref(broken))
        setattr(broken, field, 0)
        assert plan_args(p, 1, 1, 1, C.byref(broken), C.byref(n)) == 1, field
    assert lib.fa_embed_windows(p, 8, None, 0, None, 0, C.byref(seg), 4, p) == 0
    assert lib.fa_embed_windows(p, 8, None, 0, None, 1, C.byref(seg), 0, p) == 1
    bad_chunk = np.array([-1], np.int32)
    assert lib.fa_embed_windows(p, 8, None, 0, bad_chunk.ctypes.data, 1, C.byref(seg), 4, p) == 1
    assert lib.fa_weight_resample(p, 1, 0, 4, p) == 1 and lib.fa_weight_resample(p, 1, 4, 0, p) == 1
    assert lib.fa_weight_resample(None, 0, 4, 4, None) == 0 and lib.fa_weight_resample(None, 1, 4, 4, p) == 1


def test_prepare_stage_has_no_cpu_fallback(lib):
    code = (
        "import sys, numpy as np; sys.path.insert(0, %r)\n"
        "from fluidaudio_b200 import _lib\n"
        "from fluidaudio_b200.segmentation import *\n"
        "assert _lib.device_count() == 0\n"
        "seg = OfflineSegmentationProcessor()\n"
        "calls = [lambda: seg.windows(np.ones(100, np.float32)), lambda: seg.decode(np.zeros((1, 4, 7), np.float32)),\n"
        "         lambda: OfflineEmbeddingPlanner().plan(SegmentationOutput(None, np.ones((1, 4, 3), np.float32), 1, 4, 3,\n"
        "                                                np.zeros(1), 0.0), 100),\n"
        "         lambda: OfflineEmbeddingPlanner().fbank_windows(np.ones(100, np.float32), np.zeros(1)),\n"
        "         lambda: WeightInterpolation.resample([1, 2, 3], 5)]\n"
        "for call in calls:\n"
        "    try:\n"
        "        call(); raise SystemExit('ran without a device')\n"
        "    except _lib.FluidAudioError as e:\n"
        "        assert e.status == 6, str(e)\n"
        "assert seg.window_count(160001) == (6, 160000, 32000)\n"
        "print('NO_DEVICE_OK')\n" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), capture_output=True,
                         text=True, timeout=300)
    assert "NO_DEVICE_OK" in out.stdout, (out.stdout[-500:], out.stderr[-1500:])


def test_synthetic_segmentation_is_seeded_and_covers_the_cases():
    a, ta = synth.segmentation_logits(33.3, speakers=3, seed=5, frames=100)
    b, tb = synth.segmentation_logits(33.3, speakers=3, seed=5, frames=100)
    assert np.array_equal(a, b) and np.array_equal(ta["labels"], tb["labels"])
    assert a.shape == (ta["chunk_offsets"].size, 100, 7) and ta["total_samples"] == 532800
    labels = ta["labels"]
    assert (labels == 0).any() and (labels >= 4).any() and (labels[-1, 50:] == 0).all()    # silence, overlap, short tail
    assert (a.argmax(axis=2) == labels).mean() > 0.99
