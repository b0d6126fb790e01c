"""LuxTTS synthesis logic on the CPU: the Python LuxTtsSolver and the oracle against the reference's parity fixtures
(tests/golden/luxtts/), the oracle against a literal restatement (tests/luxtts_restated.py), the host build of
luxtts_core.cuh (tests/emul/luxtts_emul.cpp) against the oracle bit for bit, and fa_luxtts_plan against the oracle on
a grid that reaches every reason and boundary."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import luxtts_restated as R
from fluidaudio_b200 import _lib
from fluidaudio_b200.luxtts import LuxTtsError, LuxTtsSolver, plan as fa_plan
from oracle import oracle_luxtts as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "luxtts")
MASK = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module")
def fixtures():
    with open(os.path.join(GOLDEN, "luxtts_fixtures.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("luxtts") / "libluxtts_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(HERE, "emul", "luxtts_emul.cpp")])
    L = C.CDLL(out)
    vp, i64, u64 = C.c_void_p, C.c_int64, C.c_uint64
    L.luxtts_emul_uniform.argtypes = [u64, u64]
    L.luxtts_emul_uniform.restype = C.c_double
    L.luxtts_emul_noise.argtypes = [u64, i64, vp]
    L.luxtts_emul_step.argtypes = [vp, vp, i64, C.c_int]
    L.luxtts_emul_rms.argtypes = [vp, i64]
    L.luxtts_emul_rms.restype = C.c_float
    L.luxtts_emul_time_step.argtypes = [C.c_int]
    L.luxtts_emul_time_step.restype = C.c_double
    L.luxtts_emul_plan.argtypes = [i64, C.c_int32, C.c_int32, C.c_float, vp]
    L.luxtts_emul_plan.restype = C.c_int
    L.luxtts_emul_clip.argtypes = [C.c_float]
    L.luxtts_emul_clip.restype = C.c_float
    return L


# ------------------------------------------------------------------------------------------------ fixtures
def test_time_steps_match_the_fixture(fixtures):
    want = np.array(fixtures["solver"]["timesteps"], np.float32)
    assert np.array_equal(np.array(LuxTtsSolver.time_steps(4, 0.5), np.float32), want)
    assert np.array_equal(O.time_steps().astype(np.float32), want)
    assert O.time_steps().tolist() == LuxTtsSolver.time_steps() == R.time_steps()


def test_features_length_and_tokens_index_match_the_fixture(fixtures):
    P, pt = fixtures["prompt"]["mel_frames"], len(fixtures["prompt"]["token_ids"])
    for text in fixtures["texts"]:
        tt = len(text["token_ids"])
        assert LuxTtsSolver.features_length(P, pt, tt, 1.0) == text["features_len_speed1"]
        r = O.plan(fixtures["prompt"]["wav_24k_samples"], pt, tt, 1.0)
        assert r[0] == 0 and r[4] == text["features_len_speed1"]
        e = text["expansion"]
        assert LuxTtsSolver.tokens_index(e["tokens_len"], e["features_len"]) == e["tokens_index"]
        assert O.tokens_index(e["tokens_len"], e["features_len"]).tolist() == e["tokens_index"]
        assert len(e["tokens_index"]) == e["tokens_index_len"] and e["tokens_index"][-1] == e["tokens_len"]


def test_degenerate_duration_boundaries():
    with pytest.raises(LuxTtsError):
        LuxTtsSolver.tokens_index(10, 5)
    assert O.tokens_index(10, 5) is None and R.tokens_index(10, 5) is None
    assert LuxTtsSolver.tokens_index(4, 4) == [0, 1, 2, 3] == O.tokens_index(4, 4).tolist()


def test_mini_trajectory_matches_the_fixture(fixtures):
    s = fixtures["solver"]
    tr, ts = s["mini_trajectory"], s["timesteps"]
    x, y = np.array(tr["x0"]), np.array(tr["x0"])
    for k in range(4):
        x = LuxTtsSolver.anchor_euler_update(x, tr["v_steps"][k], ts[k], ts[k + 1], k == 3)
        y = O.anchor_euler_f64(y, tr["v_steps"][k], ts[k], ts[k + 1], k == 3)
    assert np.abs(x - np.array(tr["x_final"])).max() <= 1e-12
    assert np.abs(y - np.array(tr["x_final"])).max() <= 1e-12


def test_fixture_plan_and_rms(fixtures):
    audio = np.fromfile(os.path.join(GOLDEN, "prompt_24k_f32le.bin"), np.float32)
    assert audio.size == fixtures["prompt"]["wav_24k_samples"]
    pt = len(fixtures["prompt"]["token_ids"])
    got = [O.plan(audio.size, pt, len(t["token_ids"]), 1.0) for t in fixtures["texts"]]
    assert [g[4] for g in got] == [838, 868] and {g[6] for g in got} == {555}
    want = np.float32(fixtures["prompt"]["rms_pre_norm"])
    assert abs(int(O.rms(audio).view(np.int32)) - int(want.view(np.int32))) <= 1


# ------------------------------------------------------------------------------------------------ restatement
def test_oracle_equals_the_restatement():
    rng = np.random.default_rng(1)
    for seed in (0, 1, 42, 2**64 - 1, int(rng.integers(0, 2**63))):
        n = R.Noise(seed)
        assert O.noise(seed, 600).tobytes() == np.array([n.gaussian() for _ in range(600)], np.float32).tobytes()
    for scale in (1e-4, 0.05, 0.3):
        x = (rng.normal(size=int(rng.integers(1, 3000))) * scale).astype(np.float32)
        assert O.rms(x).tobytes() == R.rms(x).tobytes()
    x, v = rng.normal(size=500).astype(np.float32), rng.normal(size=(4, 500)).astype(np.float32)
    a, b = x, x
    for k in range(4):
        a, b = O.step(a, v[k], k), R.step(b, v[k], k)
        assert a.tobytes() == b.tobytes()
    for P, G, B in ((3, 2, 282), (50, 282, 282), (10, 555, 555)):
        xs = rng.normal(size=1024 * 100).astype(np.float32)
        assert O.vocoder_input(xs, P, G, B).tobytes() == R.vocoder_input(xs, P, G, B).tobytes()
    audio = np.concatenate([rng.normal(0, 2, 3000), [np.nan, np.inf, -np.inf, 1.0, -1.0]]).astype(np.float32)
    for r in (np.float32(0.05), np.float32(0.2)):
        for G in (2, 5, 9):
            assert O.finish(audio, G, r).tobytes() == R.finish(audio, G, r).tobytes()


# ------------------------------------------------------------------------------------------------ emulation
def _unmix(z):
    """the SplitMix64 state whose output is z (the finalizer is a bijection)"""
    z = z ^ (z >> 31) ^ (z >> 62)
    z = (z * pow(0x94D049BB133111EB, -1, 1 << 64)) & MASK
    z = z ^ (z >> 27) ^ (z >> 54)
    z = (z * pow(0xBF58476D1CE4E5B9, -1, 1 << 64)) & MASK
    return z ^ (z >> 30) ^ (z >> 60)


def test_counter_based_draws_equal_sequential_draws(emul):
    seeds = [0, 1, 42, 2**64 - 1, 0x123456789ABCDEF]
    # a seed whose first and fourth draws give z < 2^11, so u = 0 and the DBL_MIN branch runs
    seeds += [(_unmix(5) - GAMMA) & MASK, (_unmix(0) - 4 * GAMMA) & MASK]
    for seed in seeds:
        want = O.uniforms(seed, 64)
        assert [emul.luxtts_emul_uniform(seed, k + 1) for k in range(64)] == want.tolist()
    assert O.uniforms(seeds[-2], 1)[0] == 2.2250738585072014e-308
    assert O.uniforms(seeds[-1], 4)[3] == 2.2250738585072014e-308
    for seed in seeds:
        out = np.empty(2000, np.float32)
        emul.luxtts_emul_noise(seed, out.size, out.ctypes.data)
        assert out.tobytes() == O.noise(seed, out.size).tobytes()


def test_float32_update_and_rms_tree_equal_the_oracle(emul):
    rng = np.random.default_rng(2)
    x = rng.normal(size=102400).astype(np.float32)
    for k in range(4):
        v = (rng.normal(size=x.size) * 3).astype(np.float32)
        want = O.step(x, v, k)
        emul.luxtts_emul_step(x.ctypes.data, v.ctypes.data, x.size, k)
        assert x.tobytes() == want.tobytes()
    assert [emul.luxtts_emul_time_step(i) for i in range(5)] == O.time_steps().tolist()
    for n in (1, 127, 255, 256, 257, 4095, 120000):
        for scale in (1e-6, 0.01, 0.5):
            a = (rng.normal(size=n) * scale).astype(np.float32)
            assert emul.luxtts_emul_rms(a.ctypes.data, n) == O.rms(a), (n, scale)
    for v in (np.nan, np.inf, -np.inf, 2.0, -1.5, 0.25, -0.0):
        got = np.float32(emul.luxtts_emul_clip(v))
        want = O.finish(np.array([v], np.float32), 2, np.float32(1))[0]
        assert got.tobytes() == want.tobytes() or (np.isnan(got) and np.isnan(want))


# ------------------------------------------------------------------------------------------------ plan grid
SAMPLES = (0, 127, 128, 1000, 30000, 120000, 120001)
TOKENS = ((0, 5), (5, 0), (1, 1), (3, 40), (128, 127), (128, 128), (200, 55), (1, 254))
SPEEDS = (0.0, -0.0, float("nan"), float("inf"), 1e-300, 1e-45, 0.05, 0.5, 1.0, 1.3, 8.0, -1.0, 3.4e38)


def _fa(n, pt, tt, sp):
    p = fa_plan(n, pt, tt, sp)
    return (p.reason, p.prompt_samples, p.prompt_frames, p.token_count, p.features_length, p.gen_frames, p.bucket)


def test_plan_grid_equals_the_oracle_restatement_and_emulation(emul):
    seen = set()
    for n in SAMPLES:
        for pt, tt in TOKENS:
            for sp in SPEEDS:
                want = O.plan(n, pt, tt, sp)
                assert R.plan(n, pt, tt, sp) == want, (n, pt, tt, sp)
                out = np.zeros(6, np.int32)
                r = emul.luxtts_emul_plan(n, pt, tt, np.float32(sp), out.ctypes.data)
                assert (r, *out.tolist()) == want
                assert _fa(n, pt, tt, sp) == want
                seen.add(want[0])
    # genFrames 1 / 2 and buckets 282 / 283 / 555 / 556: prompt of 100 frames, 100 prompt tokens
    n = 100 * 256
    for tt, reason, bucket in ((1, 9, 0), (2, 0, 282), (282, 0, 282), (283, 0, 555), (555, 10, 0), (556, 10, 0)):
        speed = 1.0 if tt < 283 else 2.0 if tt == 283 else 1.0
        pt = 100 if tt < 283 else 50
        want = O.plan(n, pt, min(tt, 255 - pt), speed)
        assert R.plan(n, pt, min(tt, 255 - pt), speed) == want == _fa(n, pt, min(tt, 255 - pt), speed)
        seen.add(want[0])
    # exact gen boundaries through the speed: P = 100, pt = tt = 100, gen = ceil(100 / speed)
    for speed, gen in ((100.0, 1), (50.0, 2), (100 / 282, 282), (100 / 283, 283), (100 / 555, 555), (100 / 556, 556)):
        want = O.plan(n, 100, 100, speed)
        assert want == R.plan(n, 100, 100, speed) == _fa(n, 100, 100, speed)
        assert abs(want[5] - gen) <= 1   # the speed is rounded to float32 first
        seen.add(want[0])
    # degenerate: 1 prompt frame, 254 tokens -> featuresLength 1 + ceil(1 / 1 * 253) = 254 >= 254 tokens: fine;
    # with 200 / 55 at 1 frame: 1 + ceil(55 / 200) = 2 -> gen 1; a longer prompt with many prompt tokens
    want = O.plan(2 * 256, 250, 5, 1.0)   # P = 2, gen = ceil(2 / 250 * 5) = 1
    seen.add(want[0])
    want = O.plan(6 * 256, 250, 5, 0.3)   # P = 6, gen = ceil(0.4) ... = 1
    seen.add(want[0])
    want = O.plan(40 * 256, 250, 5, 0.05)   # P = 40, gen = ceil(16) = 16, L = 56 < 255 tokens
    assert want[0] == 11
    seen.add(want[0])
    assert seen >= {0, 1, 2, 3, 4, 6, 7, 8, 9, 10, 11}, seen


def test_plan_refuses_negative_counts():
    with pytest.raises(_lib.FluidAudioError):
        fa_plan(-1, 1, 1, 1.0)
