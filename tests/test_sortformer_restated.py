"""The Sortformer oracle (``oracle/oracle_sortformer.cpp``) against an independent restatement of
SortformerStateUpdater.swift (``tests/sortformer_swift.py``), bit for bit, after every update (no GPU needed).

The oracle is what the host build of ``sortformer_core.cuh`` and the GPU kernels are checked against, so a misreading
of the Swift there would pass every other test.  The restatement is written from the Swift alone, keeps the Swift's
growing arrays and both insertion sorts as written, and does every step as one float32 operation in the Swift's order.
After every update the two must agree on the confirmed and tentative rows, the whole state (speaker cache, FIFO, both
prediction arrays, the silence mean and count, the lengths), the popped rows, every stage of a compression and the next
model call's padded inputs.

Streams: every preset with every generator (synth.sortformer_chunk's four, offline-style contexts, and the adversarial
ones of ``sortformer_cases``: p exactly 0.5, exactly at the clip bounds, outside [0, 1] and subnormal, scores exactly
+0.0, fully tied scores, too few finite scores), each through at least three compressions; and every edge
configuration of ``sortformer_cases.EDGE_CONFIGS``, which must also reach the branch it is listed for.  NaN predictions
are out of scope: vDSP.clip leaves their meaning undefined.
"""
import zlib

import numpy as np
import pytest

import sortformer_cases as cases
import sortformer_swift as swift
from fluidaudio_b200.sortformer import PRESETS, SortformerConfig

D, S = 512, 4


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_sortformer
    oracle_sortformer.build()
    oracle_sortformer.lib()
    return oracle_sortformer


def same_bits(a, b, what):
    x = np.asarray(a, np.float32).reshape(-1)
    y = np.asarray(b, np.float32).reshape(-1)
    assert x.shape == y.shape, (what, x.shape, y.shape)
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), what


def check_update(ref, py):
    """everything the oracle exposes after an update equals the restatement's"""
    s, p = ref.state(), py.state
    assert (s.spkcache_length, s.fifo_length, s.silence_frames) == \
        (p.spkcacheLength, p.fifoLength, p.silenceFrameCount)
    assert (s.has_spkcache_preds, s.has_fifo_preds) == (p.spkcachePreds is not None, p.fifoPreds is not None)
    same_bits(s.spkcache, p.spkcache, "spkcache")
    same_bits(s.fifo, p.fifo, "fifo")
    same_bits(s.mean_silence, p.meanSilenceEmbedding, "meanSilenceEmbedding")
    if p.spkcachePreds is not None:
        same_bits(s.spkcache_preds, p.spkcachePreds, "spkcachePreds")
    if p.fifoPreds is not None:
        same_bits(s.fifo_preds, p.fifoPreds, "fifoPreds")
    # runMainModel's zero-padded inputs
    sc, ff, sl, fl = ref.model_inputs()
    K, F = py.config.spkcacheLen, py.config.fifoLen
    assert (sl, fl) == (p.spkcacheLength, p.fifoLength)
    same_bits(sc, np.concatenate([np.asarray(p.spkcache, np.float32), np.zeros((K - sl) * D, np.float32)]), "spkcache in")
    same_bits(ff, np.concatenate([np.asarray(p.fifo, np.float32), np.zeros((F - fl) * D, np.float32)]), "fifo in")
    # the rows the update popped, and the compression stage by stage
    pe, pp = ref.last_pop()
    if py.last_pop is None:
        assert pp.shape[0] == 0
    else:
        same_bits(pe, py.last_pop[0], "popped embeddings")
        same_bits(pp, py.last_pop[1], "popped predictions")
    comp, rec = ref.last_compression(), py.last_compression
    assert (comp is None) == (rec is None)
    if rec is not None:
        assert comp.frames == rec.frames
        for k in ("preds", "scores", "disabled", "strong", "weak"):
            same_bits(getattr(comp, k), getattr(rec, k), k)
        assert comp.indices.tolist() == rec.indices
        assert comp.is_disabled.astype(bool).tolist() == rec.is_disabled
    return comp


def run_streams(O, fields, modes, seed, max_core=0, offline=False, compressions=3):
    """each mode's stream through ``compressions`` compressions, oracle and restatement side by side; the coverage"""
    cfg, mc = SortformerConfig(**fields).resolved(max_core)
    cov = cases.Coverage()
    for mode in modes:
        rng = np.random.default_rng(seed ^ zlib.crc32(mode.encode()))
        ref, py = O.Session(fields), swift.Updater(fields)
        c = py.config
        assert ref.config == dict(chunk_len=c.chunkLen, chunk_left_context=c.chunkLeftContext,
                                  chunk_right_context=c.chunkRightContext, fifo_len=c.fifoLen,
                                  spkcache_len=c.spkcacheLen, spkcache_update_period=c.spkcacheUpdatePeriod,
                                  spkcache_sil_frames_per_spk=c.spkcacheSilFramesPerSpk)
        done = 0
        for step in range(2000):
            if done >= compressions:
                break
            n = ref.lengths()
            core, lc, rc = cases.contexts(rng, cfg, mc, ref.chunks, offline or mode == "offline")
            gen = "turns" if mode == "offline" else mode
            emb, preds = cases.chunk(rng, gen, cfg, n.spkcache_length, n.fifo_length, core, lc, rc)
            st, conf, tent = ref.update(emb, preds, lc, rc)
            assert st == 0
            pconf, ptent = py.streaming_update(emb, preds, lc, rc)
            same_bits(conf, pconf, "confirmed")
            same_bits(tent, ptent, "tentative")
            comp = check_update(ref, py)
            cov.update(cfg, n, ref.lengths(), core, comp)
            done += comp is not None
        assert done >= compressions, (mode, done)
    return cov


@pytest.mark.parametrize("name", PRESETS)
def test_presets_match_the_restatement(O, name):
    fields = vars(SortformerConfig.preset(name))
    cov = run_streams(O, fields, cases.ALL_MODES + ("offline",), zlib.crc32(name.encode()))
    print(cov.line(name))
    assert cov.c["compressions"] >= 3 * (len(cases.ALL_MODES) + 1)
    assert cov.c["ties_topk"] > 0 and cov.c["kept_neg_inf"] > 0 and cov.c["zero_scores"] > 0
    assert cov.c["half_preds"] > 0 and cov.c["at_clip_bound"] > 0


@pytest.mark.parametrize("edge", cases.EDGE_CONFIGS, ids=cases.EDGE_IDS)
def test_edge_configs_match_the_restatement(O, edge):
    cfg, _, max_core = cases.edge_config(edge)
    cov = run_streams(O, vars(cfg), edge.modes, zlib.crc32(edge.name.encode()), max_core=max_core,
                      offline=edge.offline)
    print(cov.line(edge.name))
    assert edge.reached(cov), (edge.reaches, dict(cov.c), sorted(cov.sizes))


def test_zero_scores_exist_for_every_threshold_used():
    """the CPU search finds frames with a score of exactly +0.0 and p > 0.5 for each predScoreThreshold streamed here"""
    for thr in {0.25, 0.499, 1e-6} | {e.fields.get("pred_score_threshold", 0.25) for e in cases.EDGE_CONFIGS}:
        if thr >= 0.4:   # p0 is clipped to 1 - thr: its score cannot move with p0, the search is not expected to hit
            continue
        rows = cases.zero_score_rows(thr)
        assert len(rows) > 0, thr
        for r in rows:
            s = swift.frame_scores(r, thr)[0]
            assert r[0] > 0.5 and s == 0 and not np.signbit(s)


def test_insufficient_lengths_leave_the_state_as_the_swift_does(O):
    fields = vars(SortformerConfig.preset("default"))
    rng = np.random.default_rng(8)
    ref, py = O.Session(fields), swift.Updater(fields)
    for _ in range(12):   # a FIFO with rows, so that the fifoPreds refresh runs before the throw
        n = ref.lengths()
        lc = 1 if ref.chunks else 0
        emb, preds = cases.chunk(rng, "turns", SortformerConfig(**fields), n.spkcache_length, n.fifo_length, 6, lc, 7)
        assert ref.update(emb, preds, lc, 7)[0] == 0
        py.streaming_update(emb, preds, lc, 7)
    n = ref.lengths()
    emb, preds = cases.chunk(rng, "turns", SortformerConfig(**fields), n.spkcache_length, n.fifo_length, 6, 1, 7)
    for short in (preds[:-1], preds[:n.spkcache_length + n.fifo_length + 3]):
        assert ref.update(emb, short, 1, 7)[0] == O.INSUFFICIENT_PREDS
        with pytest.raises(swift.InsufficientLength):
            py.streaming_update(emb, short, 1, 7)
        check_update(ref, py)
