"""StyleTTS2 synthesis glue on the CPU: every case of the reference's StyleTTS2GlueOpsTests and the noise-source cases
of StyleTTS2DiffusionScheduleTests against the oracle, the literal restatement (tests/styletts2_restated.py) and the
host build of styletts2_core.cuh (tests/emul/styletts2_emul.cpp); the oracle against the restatement on seeded
inputs; the host build against the oracle bit for bit, non-finite logits and features included; fa_styletts2_plan at
every bucket edge; and the façade's tail trim."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import styletts2_restated as R
from fluidaudio_b200 import _lib
from fluidaudio_b200.styletts2 import tail_trim, plan as fa_plan
from oracle import oracle_styletts2 as O

HERE = os.path.dirname(os.path.abspath(__file__))
MASK = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("styletts2") / "libstyletts2_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(HERE, "emul", "styletts2_emul.cpp")])
    L = C.CDLL(out)
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    L.styletts2_emul_bucket.argtypes = [i32, vp]
    L.styletts2_emul_noise.argtypes = [C.c_uint64, i32, vp]
    L.styletts2_emul_blend.argtypes = [vp, vp, f32, f32, vp, vp]
    L.styletts2_emul_durations.argtypes = [vp, i32, i32, vp]
    L.styletts2_emul_expand.argtypes = [vp, i32, vp, i32, vp, i32, i64, vp, vp]
    return L


def emul_durations(L, logits):
    x = np.ascontiguousarray(logits, np.float32)
    out = np.empty(x.shape[0], np.int32)
    L.styletts2_emul_durations(x.ctypes.data, x.shape[0], x.shape[1], out.ctypes.data)
    return out


def emul_expand(L, durations, d, t_en, frame_stride):
    dur = np.ascontiguousarray(durations, np.int32)
    d, t = np.ascontiguousarray(d, np.float32), np.ascontiguousarray(t_en, np.float32)
    en = np.empty((d.shape[1], frame_stride), np.float32)
    asr = np.empty((t.shape[0], frame_stride), np.float32)
    L.styletts2_emul_expand(dur.ctypes.data, dur.size, d.ctypes.data, d.shape[1], t.ctypes.data, t.shape[0],
                            frame_stride, en.ctypes.data, asr.ctypes.data)
    return en, asr


def emul_blend(L, p, r, a, b):
    p, r = np.ascontiguousarray(p, np.float32), np.ascontiguousarray(r, np.float32)
    ref, s = np.empty(128, np.float32), np.empty(128, np.float32)
    L.styletts2_emul_blend(p.ctypes.data, r.ctypes.data, float(a), float(b), ref.ctypes.data, s.ctypes.data)
    return ref, s


def bits_equal(a, b):
    """bit for bit, any NaN equal to any NaN (payloads are not compared)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and np.array_equal(np.where(both, 0, a).view(np.int32), np.where(both, 0, b).view(np.int32))


# ------------------------------------------------------------------------------------------------ StyleTTS2GlueOpsTests
def test_round_durations_clamps_at_least_one(emul):
    x = np.array([[-50.0]], np.float32)
    assert O.round_durations(x).tolist() == R.round_durations(x) == emul_durations(emul, x).tolist() == [1]


def test_round_durations_sums_sigmoid_across_channels(emul):
    x = np.zeros((2, 4), np.float32)
    assert O.round_durations(x).tolist() == R.round_durations(x) == emul_durations(emul, x).tolist() == [2, 2]


def test_build_alignment_matrix_simple():
    want = np.array([[1, 1, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0], [0, 0, 0, 1, 1, 1]], np.float32)
    m, total = O.alignment([2, 1, 3])
    assert total == 6 and np.array_equal(m, want)
    m, total = R.alignment([2, 1, 3])
    assert total == 6 and np.array_equal(m, want)


def test_build_alignment_matrix_empty():
    m, total = O.alignment([])
    assert total == 0 and m.size == 0


def test_matmul_aligned_expands_features_by_duration(emul):
    features = np.array([[1, 2, 3], [4, 5, 6]], np.float32)
    want = np.array([[1, 1, 2, 3, 3, 3], [4, 4, 5, 6, 6, 6]], np.float32)
    aln, _ = O.alignment([2, 1, 3])
    assert np.array_equal(O.matmul_aligned(features, aln), want)
    assert np.array_equal(R.matmul_aligned(features, aln), want)
    # the kernels' fused form: d = features^T (token-major) and t_en = features, both after the shift
    en, asr = emul_expand(emul, [2, 1, 3], features.T, features, 6)
    assert np.array_equal(en, O.hifigan_shift(want)) and np.array_equal(asr, O.hifigan_shift(want))


def test_transpose_last_2d():
    src = np.array([[1, 2, 3], [4, 5, 6]], np.float32)
    assert O.transpose(src).reshape(-1).tolist() == [1, 4, 2, 5, 3, 6]
    assert R.transpose(src).reshape(-1).tolist() == [1, 4, 2, 5, 3, 6]


def test_hifigan_shift_right_by_one_and_copies_column_zero():
    x = np.array([[10, 20, 30, 40], [50, 60, 70, 80]], np.float32)
    want = [10, 10, 20, 30, 50, 50, 60, 70]
    assert O.hifigan_shift(x).reshape(-1).tolist() == want == R.hifigan_shift(x).reshape(-1).tolist()


def test_hifigan_shift_single_frame_is_identity(emul):
    x = np.array([[1], [2], [3]], np.float32)
    assert np.array_equal(O.hifigan_shift(x), x) and np.array_equal(R.hifigan_shift(x), x)
    en, asr = emul_expand(emul, [1], x.T, x, 1)   # F = 1
    assert np.array_equal(en, x) and np.array_equal(asr, x)


def test_blend_style_splits_at_128_and_convex_combines(emul):
    p = np.concatenate([np.full(128, 1.0), np.full(128, 7.0)]).astype(np.float32)
    r = np.concatenate([np.full(128, 3.0), np.full(128, 9.0)]).astype(np.float32)
    for ref, s in (O.blend(p, r, 0.25, 0.75), R.blend(p, r, 0.25, 0.75), emul_blend(emul, p, r, 0.25, 0.75)):
        assert np.all(ref == np.float32(2.5)) and np.all(s == np.float32(7.5))


def test_blend_style_alpha_one_returns_diffusion_ref_half(emul):
    i = np.arange(128, dtype=np.float32)
    p = np.concatenate([i, np.full(128, -2.0, np.float32)])
    r = np.concatenate([np.full(128, -1.0, np.float32), i])
    for ref, s in (O.blend(p, r, 1.0, 0.0), R.blend(p, r, 1.0, 0.0), emul_blend(emul, p, r, 1.0, 0.0)):
        assert np.array_equal(ref, i) and np.array_equal(s, i)


# ------------------------------------------------------------------------------------------------ noise source
def test_noise_source_same_seed_equal_different_seeds_diverge(emul):
    a, b = O.noise(42, 64), O.noise(42, 64)
    assert a.tobytes() == b.tobytes()
    assert O.noise(1, 32).tobytes() != O.noise(2, 32).tobytes()
    out = np.empty(64, np.float32)
    emul.styletts2_emul_noise(42, 64, out.ctypes.data)
    assert out.tobytes() == a.tobytes()


def test_noise_source_zero_seed_is_handled(emul):
    v = O.noise(0, 8)
    assert v.size == 8 and np.any(v != 0)
    assert v.tobytes() == O.noise(0xdeadbeefcafebabe, 8).tobytes()
    out = np.empty(8, np.float32)
    emul.styletts2_emul_noise(0, 8, out.ctypes.data)
    assert out.tobytes() == v.tobytes()


def test_noise_source_gaussian_stats():
    s = O.noise(0xC0FFEE, 8192).astype(np.float64)
    mean = s.mean()
    var = ((s - np.float32(mean)) ** 2).mean()
    assert abs(mean) <= 0.1 and abs(var - 1.0) <= 0.15


def _unmix(z):
    """the SplitMix64 state whose output is z (the finalizer is a bijection)"""
    z = z ^ (z >> 31) ^ (z >> 62)
    z = (z * pow(0x94D049BB133111EB, -1, 1 << 64)) & MASK
    z = z ^ (z >> 27) ^ (z >> 54)
    z = (z * pow(0xBF58476D1CE4E5B9, -1, 1 << 64)) & MASK
    return z ^ (z >> 30) ^ (z >> 60)


def test_sampler_noise_rows_are_one_sequential_stream(emul):
    # seeds whose first / fourth draw gives u = 0 reach the DBL_MIN branch
    for seed in (0, 1, 2**64 - 1, (_unmix(5) - GAMMA) & MASK, (_unmix(0) - 4 * GAMMA) & MASK):
        tokens, mask, ni, na = O.sampler_inputs([5, 6, 7], 57, seed)
        rt, rm, rni, rna = R.sampler_inputs([5, 6, 7], 57, seed)
        assert tokens.tolist() == rt.tolist() == [5, 6, 7] + [0] * 54
        assert mask.tolist() == rm.tolist() == [1, 1, 1] + [0] * 54
        flat = np.concatenate([ni, na.reshape(-1)])
        assert flat.tobytes() == np.concatenate([rni, rna.reshape(-1)]).tobytes() == O.noise(seed, 1280).tobytes()
        out = np.empty(1280, np.float32)
        emul.styletts2_emul_noise(seed, 1280, out.ctypes.data)
        assert out.tobytes() == flat.tobytes()


# ------------------------------------------------------------------------------------------------ restatement
def test_oracle_equals_the_restatement():
    rng = np.random.default_rng(5)
    for n, c in ((1, 1), (7, 4), (40, 50)):
        logits = (rng.normal(size=(n, c)) * 4 - 1).astype(np.float32)
        dur = O.round_durations(logits)
        assert dur.tolist() == R.round_durations(logits)
        d, t_en = rng.normal(size=(n, 9)).astype(np.float32), rng.normal(size=(5, n)).astype(np.float32)
        durations, total, en, asr = O.align(logits, d, t_en)
        aln, rt = R.alignment(durations.tolist())
        assert total == rt
        assert bits_equal(en, R.hifigan_shift(R.matmul_aligned(R.transpose(d), aln)))
        assert bits_equal(asr, R.hifigan_shift(R.matmul_aligned(t_en, aln)))
    for a, b in ((0.3, 0.7), (1.0, 0.0), (0.123, -2.5)):
        p, r = rng.normal(size=256).astype(np.float32), rng.normal(size=256).astype(np.float32)
        for x, y in zip(O.blend(p, r, a, b), R.blend(p, r, a, b)):
            assert x.tobytes() == y.tobytes()
    for k in (0, 1, 50, 51, 400):
        x = rng.normal(size=k).astype(np.float32)
        assert O.trim(x).tobytes() == R.trim(x).tobytes() == tail_trim(x).tobytes()
    assert [O.bucket(n) for n in range(0, 300, 7)] == [R.bucket(n) for n in range(0, 300, 7)]


# ------------------------------------------------------------------------------------------------ emulation
SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 88.7, -88.7, 104.0, -104.0, 1e-30, 3.4e38, -3.4e38],
                   np.float32)


def test_durations_equal_the_oracle_with_non_finite_logits(emul):
    rng = np.random.default_rng(6)
    for n, c in ((1, 1), (3, 4), (256, 50), (17, 1000)):
        for scale in (0.5, 3.0, 30.0):
            logits = (rng.normal(size=(n, c)) * scale).astype(np.float32)
            want = O.round_durations(logits)
            assert emul_durations(emul, logits).tolist() == want.tolist(), (n, c, scale)
    # +-inf logits are finite sigmoids (0 and 1); any NaN traps
    x = np.array([[np.inf, -np.inf, np.inf, 0.0], [-np.inf] * 4, [88.7, -88.7, 104.0, -104.0]], np.float32)
    assert emul_durations(emul, x).tolist() == O.round_durations(x).tolist() == R.round_durations(x) == [3, 1, 2]
    for j in range(4):
        y = x.copy()
        y[1, j] = np.nan
        assert O.round_durations(y) is None and R.round_durations(y) is None
        assert emul_durations(emul, y).tolist() == [3, -1, 2]
    # sums at exact .5: 1 channel of 0 logit gives 0.5 -> rounds away from zero to 1; 3 gives 1.5 -> 2
    for c, want in ((1, 1), (3, 2), (5, 3)):
        z = np.zeros((1, c), np.float32)
        assert emul_durations(emul, z).tolist() == O.round_durations(z).tolist() == [want]


def test_expansion_equals_the_oracle_bit_for_bit(emul):
    rng = np.random.default_rng(7)
    for n, dC, tC, extra in ((1, 1, 1, 0), (3, 33, 3, 5), (60, 64, 40, 70), (200, 17, 9, 1)):
        durations = rng.integers(1, 9, size=n)
        d = rng.normal(size=(n, dC)).astype(np.float32)
        t_en = rng.normal(size=(tC, n)).astype(np.float32)
        # -0, inf and NaN in some entries: -0 becomes +0, inf and NaN reach only their own token's frames
        d.reshape(-1)[rng.choice(d.size, min(d.size, 6), replace=False)] = rng.choice(SPECIAL, min(d.size, 6))
        t_en.reshape(-1)[rng.choice(t_en.size, min(t_en.size, 6), replace=False)] = rng.choice(SPECIAL, min(t_en.size, 6))
        aln, total = O.alignment(durations)
        want_en = O.hifigan_shift(O.matmul_aligned(O.transpose(d), aln))
        want_asr = O.hifigan_shift(O.matmul_aligned(t_en, aln))
        en, asr = emul_expand(emul, durations, d, t_en, total + extra)
        assert bits_equal(en[:, :total], want_en) and bits_equal(asr[:, :total], want_asr)
        assert not en[:, total:].any() and not asr[:, total:].any()
        assert not np.signbit(en[en == 0]).any() and not np.signbit(asr[asr == 0]).any()


# ------------------------------------------------------------------------------------------------ plan
def test_plan_at_every_bucket_edge(emul):
    want = {0: (0, 1), 1: (57, 0), 57: (57, 0), 58: (64, 0), 64: (64, 0), 65: (128, 0), 128: (128, 0),
            129: (256, 0), 256: (256, 0), 257: (0, 2)}
    for n, w in want.items():
        r = C.c_int()
        assert fa_plan(n) == O.bucket(n) == R.bucket(n) == (emul.styletts2_emul_bucket(n, C.byref(r)), r.value) == w
    with pytest.raises(_lib.FluidAudioError):
        fa_plan(-1)
