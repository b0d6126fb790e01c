"""CPU checks of Sortformer's streaming state update (no GPU needed):

* the reference's two SortformerStateUpdaterTests cases on the oracle (``oracle/oracle_sortformer.cpp``) and on the
  C ABI's host-side plan (``fa_sortformer_step``);
* the configuration: the eight presets and the init's clamps;
* ``sortformer_core.cuh`` — the arithmetic the kernel runs — compiled for the host (``tests/emul/sortformer_emul.cpp``)
  against the oracle, bit for bit, compression by compression, over seeded streams of every preset;
* the host length mirror against the oracle's lengths at every step;
* the host build against the oracle over the edge configurations and adversarial predictions of ``sortformer_cases``.
"""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import sortformer_cases as cases
from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.sortformer import PRESETS, SortformerConfig, step_lengths

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# SortformerTypes.swift:121-216: chunkLen, chunkLeftContext, chunkRightContext, fifoLen, spkcacheLen, period
SWIFT_PRESETS = {
    "default": (6, 1, 7, 40, 188, 31), "fastV2": (6, 1, 7, 40, 188, 31), "fastV2_1": (6, 1, 7, 40, 188, 31),
    "balancedV2": (6, 1, 7, 188, 188, 144), "balancedV2_1": (6, 1, 7, 188, 188, 144),
    "highContextV2": (340, 1, 40, 40, 188, 300), "highContextV2_1": (340, 1, 40, 40, 188, 300),
    "efficientV2_1": (25, 1, 7, 40, 188, 31),
}
SUBSAMPLING = 8   # SortformerConfig.subsamplingFactor: coreFrames = chunkLen * 8 in the reference's tests


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_sortformer
    oracle_sortformer.build()
    oracle_sortformer.lib()
    return oracle_sortformer


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sortformer") / "libsortformer_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", "sortformer_emul.cpp")])
    L = C.CDLL(out)
    L.sortformer_emul_compress.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                           C.c_int, C.c_int] + [C.c_void_p] * 5
    L.sortformer_emul_compress.restype = None
    L.sortformer_emul_silence.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    L.sortformer_emul_silence.restype = None
    return L


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---- the reference's SortformerStateUpdaterTests ---------------------------------------------------------------------
def test_insufficient_preds_throws_and_keeps_the_state(O, lib):
    cfg = SortformerConfig.preset("default")
    core = cfg.chunk_len * SUBSAMPLING
    rows = core + cfg.chunk_left_context + cfg.chunk_right_context
    s = O.Session(vars(cfg))
    st, _, _ = s.update(np.zeros((rows, 512), np.float32), np.zeros(1, np.float32), cfg.chunk_left_context,
                        cfg.chunk_right_context)
    assert st == O.INSUFFICIENT_PREDS
    n = s.lengths()
    assert (n.spkcache_length, n.fifo_length, n.has_fifo_preds, n.has_spkcache_preds) == (0, 0, False, False)
    with pytest.raises(_lib.FluidAudioError) as e:   # one float is zero prediction rows
        step_lengths(cfg, 0, 0, False, rows, 0, cfg.chunk_left_context, cfg.chunk_right_context, max_core_frames=core)
    assert e.value.status == 1 and "insufficientPredsLength" in str(e.value)


def test_basic_flow_confirms_core_frames(O, lib):
    cfg = SortformerConfig.preset("default")
    core = cfg.chunk_len * SUBSAMPLING   # 48: more than chunkLen, so max_core must be a parameter
    rows = core + cfg.chunk_left_context + cfg.chunk_right_context
    s = O.Session(vars(cfg))
    st, conf, tent = s.update(np.zeros((rows, 512), np.float32), np.zeros((rows, 4), np.float32),
                              cfg.chunk_left_context, cfg.chunk_right_context)
    assert st == 0 and conf.size == core * 4 and tent.size == cfg.chunk_right_context * 4
    plan = step_lengths(cfg, 0, 0, False, rows, rows, cfg.chunk_left_context, cfg.chunk_right_context,
                        max_core_frames=core)
    assert plan.core == core
    n = s.lengths()
    assert (plan.spkcache_length, plan.fifo_length, plan.has_spkcache_preds) == \
        (n.spkcache_length, n.fifo_length, n.has_spkcache_preds)
    with pytest.raises(_lib.FluidAudioError):   # the default max_core (chunkLen) refuses 48 core frames
        step_lengths(cfg, 0, 0, False, rows, rows, cfg.chunk_left_context, cfg.chunk_right_context)


# ---- configuration ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PRESETS)
def test_presets_equal_the_swift_configs(lib, name):
    c = SortformerConfig.preset(name)
    chunk, lc, rc, fifo, cache, period = SWIFT_PRESETS[name]
    assert (c.chunk_len, c.chunk_left_context, c.chunk_right_context, c.fifo_len, c.spkcache_len) == \
        (chunk, lc, rc, fifo, cache)
    # the static configs go through the init: highContext's period argument 300 is held as max(min(300, 380), 340)
    assert c.spkcache_update_period == max(min(period, fifo + chunk), chunk)
    assert c.spkcache_sil_frames_per_spk == 3
    assert [np.float32(v) for v in (c.silence_threshold, c.pred_score_threshold, c.scores_boost_latest,
                                    c.strong_boost_rate, c.weak_boost_rate, c.min_pos_scores_rate)] == \
        [np.float32(v) for v in (0.2, 0.25, 0.05, 0.75, 1.5, 0.5)]
    assert c.resolved()[0] == c   # the presets are fixed points of the init's clamps


@pytest.mark.parametrize("fields", [
    dict(chunk_len=0), dict(chunk_len=-3, spkcache_update_period=0), dict(spkcache_len=4),
    dict(spkcache_len=10, spkcache_sil_frames_per_spk=5), dict(spkcache_update_period=1000),
    dict(spkcache_update_period=2, chunk_len=9), dict(fifo_len=0, spkcache_update_period=100),
])
def test_config_clamps(O, lib, fields):
    cfg = SortformerConfig(**fields)
    got, max_core = cfg.resolved()
    sil = cfg.spkcache_sil_frames_per_spk
    chunk = max(1, cfg.chunk_len)
    assert got.chunk_len == chunk and max_core == chunk
    assert got.spkcache_len == max(cfg.spkcache_len, (1 + sil) * 4)
    assert got.spkcache_update_period == max(min(cfg.spkcache_update_period, cfg.fifo_len + chunk), chunk)
    ref = O.Session(vars(cfg)).config
    assert all(ref[k] == getattr(got, k) for k in ref)


@pytest.mark.parametrize("fields, max_core", [
    (dict(fifo_len=-1), 0), (dict(chunk_left_context=-1), 0), (dict(spkcache_sil_frames_per_spk=-1), 0),
    (dict(silence_threshold=float("nan")), 0), (dict(weak_boost_rate=float("inf")), 0),
    (dict(spkcache_len=20000, fifo_len=5000), 0), (dict(), 24999 - 188 - 40 - 3 + 1),
])
def test_config_rejections(lib, fields, max_core):
    with pytest.raises(_lib.FluidAudioError) as e:
        SortformerConfig(**fields).resolved(max_core)
    assert e.value.status == 1
    SortformerConfig().resolved(24999 - 188 - 40 - 3)   # (188 + 40 + max_core + 3) * 4 = 99 996 < maxIndex


# ---- emulation of the kernel's arithmetic and the host mirror against the oracle -------------------------------------
def stream_contexts(cfg, chunks, offline, rng):
    """(core, lc, rc) per chunk: the streaming rule, or offline-style contexts with a short last chunk"""
    out = []
    for i in range(chunks):
        lc = cfg.chunk_left_context if i > 0 else 0
        rc, core = cfg.chunk_right_context, cfg.chunk_len
        if offline and i == chunks - 1:
            core, rc = max(1, cfg.chunk_len // 2), int(rng.integers(0, cfg.chunk_right_context + 1))
        out.append((core, lc, rc))
    return out


def chunk_count(cfg, compressions=3):
    """chunks for at least `compressions` compressions of a stream"""
    first = cfg.spkcache_len + cfg.fifo_len + cfg.spkcache_update_period
    return -(-(first + (compressions - 1) * cfg.spkcache_update_period) // cfg.chunk_len) + 2


def run_emulated(emul, cfg, K, comp):
    L = comp.frames
    res = [np.zeros((L, 4), np.float32) for _ in range(4)]
    slot = np.zeros(K, np.int32)
    c, _ = cfg.resolved()
    per = c.spkcache_len // 4 - c.spkcache_sil_frames_per_spk
    k = lambda r: int(np.float32(per) * np.float32(r))
    pr = np.ascontiguousarray(comp.preds)
    emul.sortformer_emul_compress(pr.ctypes.data, L, K, c.spkcache_sil_frames_per_spk, c.pred_score_threshold,
                                  c.scores_boost_latest, k(c.strong_boost_rate), k(c.weak_boost_rate),
                                  k(c.min_pos_scores_rate), *[r.ctypes.data for r in res], slot.ctypes.data)
    return res, slot


@pytest.mark.parametrize("name", PRESETS)
@pytest.mark.parametrize("mode", synth.SORTFORMER_MODES + ("offline",))
def test_emulation_and_mirror_match_the_oracle(O, lib, emul, name, mode):
    cfg = SortformerConfig.preset(name)
    rng = np.random.default_rng(zlib.crc32(f"{name}/{mode}".encode()))
    s = O.Session(vars(cfg))
    K = cfg.spkcache_len
    lengths = (0, 0, False)
    mean, count = np.zeros(512, np.float32), np.zeros(1, np.int64)
    compressions = 0
    for core, lc, rc in stream_contexts(cfg, chunk_count(cfg), mode == "offline", rng):
        n = s.lengths()
        gen = "turns" if mode == "offline" else mode
        emb, preds = synth.sortformer_chunk(rng, gen, n.spkcache_length, n.fifo_length, core, lc, rc)
        plan = step_lengths(cfg, *lengths, emb.shape[0], preds.shape[0], lc, rc)
        st, _, _ = s.update(emb, preds, lc, rc)
        assert st == 0
        n = s.lengths()
        lengths = (plan.spkcache_length, plan.fifo_length, plan.has_spkcache_preds)
        assert lengths == (n.spkcache_length, n.fifo_length, n.has_spkcache_preds)
        pop_e, pop_p = s.last_pop()
        assert plan.pop == pop_p.shape[0]
        emul.sortformer_emul_silence(pop_e.ctypes.data, pop_p.ctypes.data, pop_p.shape[0], cfg.silence_threshold,
                                     mean.ctypes.data, count.ctypes.data)
        assert np.array_equal(bits(mean), bits(s.state().mean_silence)) and count[0] == n.silence_frames
        comp = s.last_compression()
        assert plan.compress == (comp is not None)
        if comp is None:
            continue
        compressions += 1
        (sc, dis, strong, weak), slot = run_emulated(emul, cfg, K, comp)
        for got, ref in ((sc, comp.scores), (dis, comp.disabled), (strong, comp.strong), (weak, comp.weak)):
            assert np.array_equal(bits(got), bits(ref))
        assert np.array_equal(slot < 0, comp.is_disabled.astype(bool))
        assert np.array_equal(slot[slot >= 0], comp.indices[slot >= 0])
    assert compressions >= 3
    if mode == "silence":
        assert count[0] > 0
    if mode == "never_silent":
        assert count[0] == 0 and not mean.any()


@pytest.mark.parametrize("edge", cases.EDGE_CONFIGS, ids=cases.EDGE_IDS)
def test_emulation_matches_the_oracle_on_edge_configs(O, lib, emul, edge):
    """the host build against the oracle over the edge configurations, every generator including the adversarial
    ones, compression by compression"""
    cfg, resolved, max_core = cases.edge_config(edge)
    K = resolved.spkcache_len
    for mode in edge.modes:
        rng = np.random.default_rng(zlib.crc32(f"{edge.name}/{mode}".encode()))
        s = O.Session(vars(cfg))
        mean, count = np.zeros(512, np.float32), np.zeros(1, np.int64)
        compressions = 0
        while compressions < 3:
            assert s.chunks < 2000
            n = s.lengths()
            core, lc, rc = cases.contexts(rng, resolved, max_core, s.chunks, edge.offline)
            emb, preds = cases.chunk(rng, mode, resolved, n.spkcache_length, n.fifo_length, core, lc, rc)
            assert s.update(emb, preds, lc, rc)[0] == 0
            pop_e, pop_p = s.last_pop()
            emul.sortformer_emul_silence(pop_e.ctypes.data, pop_p.ctypes.data, pop_p.shape[0],
                                         resolved.silence_threshold, mean.ctypes.data, count.ctypes.data)
            assert np.array_equal(bits(mean), bits(s.state().mean_silence)) and count[0] == s.lengths().silence_frames
            comp = s.last_compression()
            if comp is None:
                continue
            compressions += 1
            (sc, dis, strong, weak), slot = run_emulated(emul, cfg, K, comp)
            for got, ref in ((sc, comp.scores), (dis, comp.disabled), (strong, comp.strong), (weak, comp.weak)):
                assert np.array_equal(bits(got), bits(ref))
            assert np.array_equal(slot < 0, comp.is_disabled.astype(bool))
            assert np.array_equal(slot[slot >= 0], comp.indices[slot >= 0])
