"""Offline Sortformer windows on the CPU: the reference's OfflineSortformerTests stitcher cases and config defaults
against the oracle (oracle/oracle_offline_sortformer.cpp), the literal restatement (tests/offline_sortformer_restated.py)
and the host build of offline_sortformer_core.cuh (tests/emul/offline_sortformer_emul.cpp); the oracle against the
restatement on whole files; the host build against the oracle bit for bit on random and adversarial predictions at
every overlap; and fa_offline_sortformer_plan at every frame and overlap edge."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import offline_sortformer_cases as K
import offline_sortformer_restated as R
from fluidaudio_b200 import _lib
from fluidaudio_b200.offline_sortformer import OfflineSortformerConfig, OfflineSortformerWindows
from oracle import oracle_offline_sortformer as O

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("offline_sortformer") / "libosf_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(HERE, "emul", "offline_sortformer_emul.cpp")])
    L = C.CDLL(out)
    vp, i32, i64 = C.c_void_p, C.c_int, C.c_int64
    L.osf_emul_clamp.argtypes = [i32]
    L.osf_emul_plan.argtypes = [i32, i64, vp, vp]
    L.osf_emul_perm.argtypes = [i32, i32]
    L.osf_emul_alignment.argtypes = [vp, vp, i32, vp]
    L.osf_emul_stitch.argtypes = [i32, i64, vp, vp, vp]
    return L


def emul_alignment(L, g, w, frames):
    g, w = np.ascontiguousarray(g, np.float32), np.ascontiguousarray(w, np.float32)
    out = np.empty(4, np.int32)
    L.osf_emul_alignment(g.ctypes.data, w.ctypes.data, int(frames), out.ctypes.data)
    return out.tolist()


def emul_stitch(L, overlap, frames, preds):
    windows, total = R.plan(frames, overlap)
    p = np.ascontiguousarray(preds, np.float32)
    assert p.shape == (windows, 384, 4)
    out, maps = np.full((total, 4), 7, np.float32), np.empty((windows, 4), np.int32)
    L.osf_emul_stitch(int(overlap), int(frames), p.ctypes.data, out.ctypes.data, maps.ctypes.data)
    return out, maps


def oracle_stitch(overlap, frames, preds):
    """the oracle's loop with a model that returns window k's preset predictions on its k-th call"""
    calls = iter(np.asarray(preds, np.float32))
    return O.stitch(np.zeros((int(frames), 128), np.float32), frames, overlap, lambda mel, ml: next(calls))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same_bits(a, b):
    """bit for bit, any NaN equal to any NaN (payloads are not compared)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and np.array_equal(bits(np.where(both, 0, a)), bits(np.where(both, 0, b)))


# ------------------------------------------------------------------------------------------------ OfflineSortformerTests
def _three(emul, g, w, frames):
    got = [O.alignment(g, w, frames), R.alignment(g, w, frames), emul_alignment(emul, g, w, frames)]
    assert got[0] == got[1] == got[2], got
    return got[0]


def test_stitcher_identity_when_aligned(emul):
    g = np.zeros(16, np.float32)
    for f in range(4):
        g[f * 4 + f % 4] = 1
    assert _three(emul, g, g.copy(), 4) == [0, 1, 2, 3]


def test_stitcher_recovers_permutation(emul):
    perm = [2, 0, 3, 1]
    g, w = np.zeros(32, np.float32), np.zeros(32, np.float32)
    for f in range(8):
        g[f * 4 + f % 4] = 1
        w[f * 4 + perm[f % 4]] = 1
    mapping = _three(emul, g, w, 8)
    for f in range(8):
        for c in range(4):
            if w[f * 4 + c] > 0:
                assert mapping[c] == f % 4


def test_stitcher_soft_activity(emul):
    g, w = np.full(12, 0.1, np.float32), np.full(12, 0.1, np.float32)
    for f in range(3):
        g[f * 4 + 1] = 0.9
        w[f * 4 + 3] = 0.9
    assert _three(emul, g, w, 3)[3] == 1


def test_stitcher_zero_frames_is_identity(emul):
    assert _three(emul, np.zeros(4, np.float32), np.zeros(4, np.float32), 0) == [0, 1, 2, 3]


def test_stitcher_mapping_is_bijection(emul):
    g, w = np.zeros(20, np.float32), np.zeros(20, np.float32)
    for f in range(5):
        g[f * 4 + f % 4] = f + 1
        w[f * 4 + (f + 2) % 4] = f + 1
    assert sorted(_three(emul, g, w, 5)) == [0, 1, 2, 3]


def test_offline_config_defaults(emul):
    cfg = OfflineSortformerConfig.offline_v2_1()
    assert (cfg.window_output_frames, cfg.subsampling_factor, cfg.window_mel_frames, cfg.num_speakers,
            cfg.overlap_output_frames, cfg.mel_features) == (384, 8, 3072, 4, 100, 128)
    assert np.float32(cfg.frame_duration_seconds) == R.frame_duration_seconds() == np.float32(0.08)
    assert abs(cfg.frame_duration_seconds - 0.08) < 1e-6
    assert [emul.osf_emul_clamp(v) for v in K.OVERLAP_EDGES] == [R.clamp_overlap(v) for v in K.OVERLAP_EDGES] == \
        [0, 0, 1, 100, 383, 383, 383]


def test_permutation_order_is_the_swap_recursion(emul):
    want = ("0123 0132 0213 0231 0321 0312 1023 1032 1203 1230 1320 1302 2103 2130 2013 2031 2301 2310 3120 3102 "
            "3210 3201 3021 3012").split()
    assert ["".join(map(str, p)) for p in R.permutations()] == want
    assert ["".join(str(emul.osf_emul_perm(p, g)) for g in range(4)) for p in range(24)] == want


# ------------------------------------------------------------------------------------------------ oracle vs restatement
@pytest.mark.parametrize("overlap", [100, 0, 383, 1])
def test_oracle_matches_the_restatement_on_whole_files(overlap):
    rng = np.random.default_rng(overlap + 3)
    for frames in (1, 3001, 3072, 3073, 5344):
        rows = K.mel_rows(rng, frames)
        if overlap == 383 and frames > 3073:
            continue   # 18 windows of Python arithmetic; the edge is covered at 3073
        og, om = O.stitch(rows, frames, overlap, K.model)
        rg, rm = R.stitch(rows, frames, overlap, K.model)
        assert same_bits(og, rg) and np.array_equal(om, rm), (frames, overlap)


def test_oracle_matches_the_restatement_on_adversarial_overlaps():
    rng = np.random.default_rng(12)
    for kind in K.KINDS:
        for ov in (1, 2, 7, 100):
            g = K.adversarial_preds(rng, 1, kind)[0, :ov]
            w = K.adversarial_preds(rng, 1, kind)[0, :ov]
            assert O.alignment(g, w, ov) == R.alignment(g, w, ov), (kind, ov)


# ------------------------------------------------------------------------------------------------ host build vs oracle
@pytest.mark.parametrize("kind", K.KINDS)
def test_emulation_matches_the_oracle_alignment(emul, kind):
    rng = np.random.default_rng(hash(kind) & 0xffff)
    for ov in list(range(1, 12)) + [31, 100, 255, 382, 383]:
        g = K.adversarial_preds(rng, 1, kind)[0, :ov]
        w = K.adversarial_preds(rng, 1, kind)[0, :ov]
        assert emul_alignment(emul, g, w, ov) == O.alignment(g, w, ov), (kind, ov)
    if kind == "nan":
        assert emul_alignment(emul, g, w, 383) == [0, 1, 2, 3]


def test_tied_and_signed_zero_scores_keep_the_first():
    # every correlation +0 or -0: all scores tie at zero, identity (the first) keeps the lead
    g = np.array([[1, 1, 1, 1]], np.float32)
    w = np.array([[0.0, -0.0, 0.0, -0.0]], np.float32)
    assert O.alignment(g, w, 1) == R.alignment(g, w, 1) == [0, 1, 2, 3]
    # -inf scores never beat -FLT_MAX, +inf wins
    w = np.array([[-np.inf, -np.inf, -np.inf, -np.inf]], np.float32)
    assert O.alignment(g, w, 1) == [0, 1, 2, 3]
    g, w = np.array([[1, 0, 0, 0]], np.float32), np.array([[0, np.inf, 0, 0]], np.float32)
    assert O.alignment(g, w, 1) == R.alignment(g, w, 1) == [1, 0, 2, 3]


@pytest.mark.parametrize("kind", K.KINDS)
@pytest.mark.parametrize("overlap", [1, 2, 100, 200, 383])
def test_emulation_matches_the_oracle_stitch(emul, kind, overlap):
    rng = np.random.default_rng(overlap * 7 + len(kind))
    for frames in (1, 3001, 3072, 3073, 5344, 9000):
        windows, _ = R.plan(frames, overlap)
        preds = K.adversarial_preds(rng, windows, kind)
        eg, em = emul_stitch(emul, overlap, frames, preds)
        og, om = oracle_stitch(overlap, frames, preds)
        assert same_bits(eg, og) and np.array_equal(em, om), (frames, overlap, kind)
        if kind == "nan":
            assert (om == np.arange(4)).all()


# ------------------------------------------------------------------------------------------------ plan
@pytest.mark.parametrize("overlap", K.OVERLAP_EDGES)
def test_plan_matches_the_restatement(emul, overlap):
    frames = [0, *K.FRAME_EDGES, K.HOUR, 2272 * 5 + 3072, 2272 * 5 + 3073, 12345, 40000]
    w, r = OfflineSortformerWindows().plan(frames, overlap)
    want = [R.plan(n, overlap) for n in frames]
    assert list(zip(w.tolist(), r.tolist())) == want
    for n, (ww, rr) in zip(frames, want):
        a, b = C.c_int64(), C.c_int64()
        emul.osf_emul_plan(overlap, n, C.byref(a), C.byref(b))
        assert (a.value, b.value) == (ww, rr)


def test_plan_worked_values():
    w, r = OfflineSortformerWindows().plan([1, 3001, 3072, 3073, 5344, K.HOUR, 0], 100)
    assert w.tolist() == [1, 1, 2, 2, 3, 159, 0] and r.tolist() == [1, 376, 384, 385, 668, 45001, 0]


def test_plan_refuses_a_negative_frame_count():
    L = _lib.load()
    n = np.array([5, -1], np.int64)
    w, r = np.full(2, -9, np.int64), np.full(2, -9, np.int64)
    assert L.fa_offline_sortformer_plan(100, 2, n.ctypes.data, w.ctypes.data, r.ctypes.data) == 1
    assert (w == -9).all() and (r == -9).all() and b"mel_frames[1]" in L.fa_last_error()
