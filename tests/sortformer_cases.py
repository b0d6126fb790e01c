"""Shared pieces of the Sortformer state tests (not a test module):

* ``EDGE_CONFIGS``: configurations that fa_sortformer_resolve_config accepts, each aimed at one branch of
  SortformerStateUpdater.swift, with a check that the init's clamps kept the edge and a check that a stream reached it;
* ``chunk``: the model outputs of one update, from synth.sortformer_chunk's generators or the adversarial ones here;
* ``Coverage``: what a stream reached (pops by kind, compressions, ties decided by index, kept -inf slots, ...);
* ``Harness``: a SortformerStreams handle driven against one oracle session per device session.

NaN predictions are out of scope everywhere: vDSP.clip leaves their meaning undefined.
"""
from __future__ import annotations

import collections
import functools
import zlib
from types import SimpleNamespace

import numpy as np

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams

import sortformer_swift as swift

D, S = 512, 4
F32 = np.float32
LN2 = float(np.log(2.0))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def chunks_needed(cfg, compressions=3):
    first = cfg.spkcache_len + cfg.fifo_len + cfg.spkcache_update_period
    return -(-(first + (compressions - 1) * cfg.spkcache_update_period) // cfg.chunk_len) + 2


def k_values(cfg):
    """(strong, weak, minPos) per speaker of a resolved config (SortformerStateUpdater.swift:229-232)"""
    per = cfg.spkcache_len // S - cfg.spkcache_sil_frames_per_spk
    return tuple(int(F32(per) * F32(r)) for r in (cfg.strong_boost_rate, cfg.weak_boost_rate, cfg.min_pos_scores_rate))


# ---- adversarial predictions -----------------------------------------------------------------------------------------
ADVERSARIAL_MODES = ("half", "bounds", "extremes", "zero_score", "constant", "sparse")
ALL_MODES = synth.SORTFORMER_MODES + ADVERSARIAL_MODES
NONNEGATIVE_MODES = tuple(m for m in ALL_MODES if m != "extremes")   # every probability in [0, 1]
EXTREMES = np.array([0.0, -0.0, 1.0, 0.5, -0.25, -3.0, 1.25, 7.0, 1e-40, -1e-40, 1.4e-45, 0.999999], np.float32)


@functools.lru_cache(maxsize=None)
def zero_score_rows(threshold: float, want: int = 24):
    """Frames [n x 4] whose speaker-0 score (getLogPredScores) is exactly +0.0 with p0 > 0.5, found by a CPU search
    over float32 inputs with the restatement's score function: other speakers drawn at random, p0 scanned over the
    consecutive float32 values around the real root p0 = 0.5 / prod(1 - p_other).  A -0.0 score cannot occur: the last
    operation adds the frame's log1p sum, which starts from +0.0 and so is never -0.0, and x + y is -0.0 under round to
    nearest only when both are -0.0."""
    thr = F32(threshold)
    rng = np.random.default_rng(zlib.crc32(np.float32(threshold).tobytes()))
    found = []
    for _ in range(400):
        others = rng.uniform(0.0, 0.45, size=3).astype(np.float32)
        root = 0.5 / float(np.prod(1.0 - others.astype(np.float64)))
        if not 0.5 < root < 1.0:
            continue
        centre = np.float32(root).view(np.int32)
        for p0 in (centre + np.arange(-64, 65, dtype=np.int32)).view(np.float32):
            row = np.array([p0, *others], np.float32)
            s = swift.frame_scores(row, thr)[0]
            if p0 > 0.5 and s == 0:
                assert not np.signbit(s)
                found.append(row)
                break
        if len(found) >= want:
            break
    return np.array(found, np.float32).reshape(-1, S)


def _mix(rng, p, values, share=0.3):
    """p with about ``share`` of its entries replaced by draws from ``values``"""
    m = rng.random(p.shape) < share
    p[m] = rng.choice(np.asarray(values, np.float32), size=int(m.sum()))
    return p


def chunk(rng, mode, cfg, spkcache_length, fifo_length, core, lc, rc):
    """One model output (chunk embeddings [lc + core + rc x 512], probabilities [spkcache + fifo + lc + core + rc x 4])
    of a ``mode`` stream.  synth.sortformer_chunk's modes, and:

    ``half``: p exactly 0.5 (disabled: p <= 0.5); ``bounds``: p exactly thr and 1 - thr (the clip bounds);
    ``extremes``: 0, -0, 1, negatives, values above 1 and subnormals; ``zero_score``: frames whose score is exactly +0.0
    with p > 0.5 (disabled only when the speaker has enough positive scores); ``constant``: one probability for every
    frame and speaker, so every score ties and only the index decides; ``sparse``: nearly all frames silent, so fewer
    finite scores than spkcacheLen remain and -inf entries are kept (maxIndex slots)."""
    if mode in synth.SORTFORMER_MODES:
        return synth.sortformer_chunk(rng, mode, spkcache_length, fifo_length, core, lc, rc)
    rows = spkcache_length + fifo_length + lc + core + rc
    emb = rng.normal(0.0, 1.0, size=(lc + core + rc, D)).astype(np.float32)
    thr = F32(cfg.pred_score_threshold)
    if mode == "constant":
        # one value for every row of a call: 0.75 (every score ties), on about one call in five 0.3 (all disabled)
        v = F32(0.3) if rng.random() < 0.2 else F32(0.75)
        return emb, np.full((rows, S), v, np.float32)
    if mode == "sparse":
        p = rng.uniform(0.0, 0.2, size=(rows, S)).astype(np.float32)
        hit = rng.random(rows) < 0.04
        p[hit, rng.integers(0, S, size=int(hit.sum()))] = rng.uniform(0.6, 1.0, size=int(hit.sum()))
        return emb, p
    _, p = synth.sortformer_chunk(rng, "turns", spkcache_length, fifo_length, core, lc, rc)
    if mode == "half":
        return emb, _mix(rng, p, [0.5])
    if mode == "bounds":
        return emb, _mix(rng, p, [thr, F32(1) - thr])
    if mode == "extremes":
        return emb, _mix(rng, p, EXTREMES, 0.2)
    if mode == "zero_score":
        z = zero_score_rows(float(thr))
        if len(z):
            m = rng.random(rows) < 0.35
            p[m] = z[rng.integers(0, len(z), size=int(m.sum()))]
        return emb, p
    raise ValueError(mode)


# ---- edge configurations ---------------------------------------------------------------------------------------------
SMALL = dict(chunk_len=6, chunk_left_context=1, chunk_right_context=3, fifo_len=10, spkcache_len=24,
             spkcache_update_period=8, spkcache_sil_frames_per_spk=1)


def _edge(name, reaches, fields, kept=lambda c, m: True, reached=lambda v: True, max_core=0, modes=ALL_MODES,
          offline=False):
    """``kept(resolved, max_core)``: the edge survived the init's clamps; ``reached(coverage)``: a stream reached it;
    ``offline``: some chunks are short (core < chunkLen) or, with max_core above chunkLen, long"""
    return SimpleNamespace(name=name, reaches=reaches, fields={**SMALL, **fields}, kept=kept, reached=reached,
                           max_core=max_core, modes=modes, offline=offline)


def _n_edge(chunk_len):
    # fifoLen 0 pops every core frame: after the first compression L = 40 + chunk_len, N = (L + 2) * 4
    n = (40 + chunk_len + 2) * S
    return _edge(f"N{n}", f"compression over N = {n} permuted scores ({n % 256:+d} past a multiple of 256 threads)",
                 dict(fifo_len=0, spkcache_len=40, spkcache_sil_frames_per_spk=2, chunk_len=chunk_len,
                      chunk_right_context=1),
                 kept=lambda c, m: c.fifo_len == 0 and c.spkcache_len == 40, reached=lambda v: n in v.sizes)


EDGE_CONFIGS = [
    _edge("fifo0", "fifoLen 0: every core frame pops straight into the cache; fifoPreds never refreshed",
          dict(fifo_len=0, spkcache_update_period=3),
          kept=lambda c, m: c.fifo_len == 0 and c.spkcache_update_period == c.chunk_len,
          reached=lambda v: v.c["fifo_refresh"] == 0 and v.c["pop_period"] > 0),
    _edge("period_below_chunk", "period below chunkLen is raised to chunkLen: pop = chunkLen",
          dict(chunk_len=8, spkcache_update_period=3), kept=lambda c, m: c.spkcache_update_period == 8,
          reached=lambda v: v.c["pop_period"] > 0),
    _edge("period_equal_chunk", "period equal to chunkLen", dict(chunk_len=8, spkcache_update_period=8),
          kept=lambda c, m: c.spkcache_update_period == 8, reached=lambda v: v.c["pop_period"] > 0),
    _edge("period_above_chunk", "period between chunkLen and fifoLen + chunkLen",
          dict(fifo_len=20, spkcache_update_period=13),
          kept=lambda c, m: c.spkcache_update_period == 13, reached=lambda v: v.c["pop_period"] > 0),
    _edge("period_above_context", "period above fifoLen + chunkLen is lowered to it; short chunks pop the whole "
          "context (min(pop, contextLength))", dict(spkcache_update_period=100),
          kept=lambda c, m: c.spkcache_update_period == c.fifo_len + c.chunk_len,
          reached=lambda v: v.c["pop_context"] > 0, offline=True),
    _edge("overflow_above_period", "long chunks overflow the FIFO by more than the period: pop = the overflow",
          dict(spkcache_update_period=6), max_core=20, kept=lambda c, m: m == 20 and c.spkcache_update_period == 6,
          reached=lambda v: v.c["pop_overflow"] > 0, offline=True),
    _edge("sil0", "spkcacheSilFramesPerSpk 0: no placeholders", dict(spkcache_sil_frames_per_spk=0),
          kept=lambda c, m: c.spkcache_sil_frames_per_spk == 0, reached=lambda v: v.c["compressions"] >= 3),
    _edge("per_spk_one_all_k_zero", "spkcacheLen 5 with 6 silence frames: the init raises spkcacheLen to 28, so "
          "spkcacheLenPerSpk stays 1 (it cannot reach 0); rates below 1 make every k 0: no boosts, and minPos 0 "
          "disables every non-positive score",
          dict(spkcache_len=5, spkcache_sil_frames_per_spk=6, weak_boost_rate=0.5),
          kept=lambda c, m: c.spkcache_len == 28 and k_values(c) == (0, 0, 0),
          reached=lambda v: v.c["strong_none"] == v.c["weak_none"] == v.c["compressions"] > 0
          and v.c["nonpos_disabled"] > 0 and v.c["nonpos_kept"] == 0),
    _edge("cache5", "spkcacheLen 5, not a multiple of 4", dict(spkcache_len=5, spkcache_sil_frames_per_spk=0),
          kept=lambda c, m: c.spkcache_len == 5, reached=lambda v: v.c["compressions"] >= 3),
    _edge("cache13", "spkcacheLen 13, not a multiple of 4", dict(spkcache_len=13),
          kept=lambda c, m: c.spkcache_len == 13, reached=lambda v: v.c["compressions"] >= 3),
    _edge("boost_rates_zero", "strong and weak rate 0: k = 0, no boost",
          dict(strong_boost_rate=0.0, weak_boost_rate=0.0), kept=lambda c, m: k_values(c)[:2] == (0, 0),
          reached=lambda v: v.c["strong_none"] == v.c["weak_none"] == v.c["compressions"] > 0),
    _edge("boost_rates_large", "strong and weak k above the cache length: every finite score is boosted",
          dict(strong_boost_rate=40.0, weak_boost_rate=64.0), kept=lambda c, m: min(k_values(c)[:2]) >= 200,
          reached=lambda v: v.c["strong_all"] > 0 and v.c["weak_all"] > 0 and v.c["strong_some"] == 0),
    _edge("min_pos_zero", "minPosScoresRate 0: every non-positive score is disabled", dict(min_pos_scores_rate=0.0),
          kept=lambda c, m: k_values(c)[2] == 0,
          reached=lambda v: v.c["nonpos_disabled"] > 0 and v.c["nonpos_kept"] == 0),
    _edge("min_pos_one", "minPosScoresRate 1: non-positive scores kept until a speaker has perSpk positive ones",
          dict(min_pos_scores_rate=1.0), kept=lambda c, m: k_values(c)[2] == 5,
          reached=lambda v: v.c["nonpos_kept"] > 0),
    _edge("min_pos_above_one", "minPosScoresRate 3: no speaker reaches minPos, no non-positive score disabled",
          dict(min_pos_scores_rate=3.0), kept=lambda c, m: k_values(c)[2] == 15,
          reached=lambda v: v.c["nonpos_kept"] > 0 and v.c["nonpos_disabled"] == 0),
    _edge("latest_zero", "scoresBoostLatest 0", dict(scores_boost_latest=0.0),
          kept=lambda c, m: c.scores_boost_latest == 0, reached=lambda v: v.c["latest_scored"] > 0),
    _edge("latest_negative", "scoresBoostLatest -6: recent frames lose to older ones they beat",
          dict(scores_boost_latest=-6.0, strong_boost_rate=0.0, weak_boost_rate=0.0),
          kept=lambda c, m: c.scores_boost_latest < 0,
          reached=lambda v: v.c["latest_reorder"] > 0),
    _edge("latest_large", "scoresBoostLatest 50: recent frames win over older ones they lose to",
          dict(scores_boost_latest=50.0, strong_boost_rate=0.0, weak_boost_rate=0.0),
          kept=lambda c, m: c.scores_boost_latest == 50,
          reached=lambda v: v.c["latest_reorder"] > 0),
    _edge("threshold_near_zero", "predScoreThreshold 1e-6: clip bounds 1e-6 and 1 - 1e-6",
          dict(pred_score_threshold=1e-6), kept=lambda c, m: 0 < c.pred_score_threshold < 1e-5,
          reached=lambda v: v.c["at_clip_bound"] > 0),
    _edge("threshold_near_half", "predScoreThreshold 0.499: clip bounds 0.499 and 0.501",
          dict(pred_score_threshold=0.499), kept=lambda c, m: abs(c.pred_score_threshold - 0.499) < 1e-6,
          reached=lambda v: v.c["at_clip_bound"] > 0),
    _edge("silence_zero", "silenceThreshold 0: no frame is silent", dict(silence_threshold=0.0),
          kept=lambda c, m: c.silence_threshold == 0, reached=lambda v: v.c["popped"] > 0 and v.c["silent"] == 0,
          modes=NONNEGATIVE_MODES),
    _edge("silence_four", "silenceThreshold 4.5: every frame is silent", dict(silence_threshold=4.5),
          kept=lambda c, m: c.silence_threshold == 4.5,
          reached=lambda v: v.c["popped"] > 0 and v.c["silent"] == v.c["popped"], modes=NONNEGATIVE_MODES),
    _n_edge(10), _n_edge(21), _n_edge(22), _n_edge(23), _n_edge(85), _n_edge(86), _n_edge(87),
]
EDGE_IDS = [e.name for e in EDGE_CONFIGS]


def edge_config(e):
    """(SortformerConfig, resolved config, resolved max_core), asserting the edge survived the init's clamps"""
    cfg = SortformerConfig(**e.fields)
    resolved, max_core = cfg.resolved(e.max_core)
    assert e.kept(resolved, max_core), (e.name, resolved, max_core)
    return cfg, resolved, max_core


def contexts(rng, cfg, max_core, chunks_done, offline):
    """(core, lc, rc) of a session's next update: the streaming rule, and with ``offline`` now and then a short chunk,
    or a long one when max_core is above chunkLen"""
    lc = cfg.chunk_left_context if chunks_done > 0 else 0
    core, rc = cfg.chunk_len, cfg.chunk_right_context
    if offline and rng.random() < 0.4:
        core = int(rng.integers(1, max(max_core, cfg.chunk_len) + 1))
        rc = int(rng.integers(0, cfg.chunk_right_context + 1))
    return core, lc, rc


# ---- coverage --------------------------------------------------------------------------------------------------------
class Coverage:
    """What a set of streams reached, counted from the oracle's lengths and compression stages."""

    def __init__(self):
        self.c = collections.Counter()
        self.sizes = set()

    def update(self, cfg, before, after, core, comp):
        """one update: the lengths before and after (oracle_sortformer lengths()), its core frames and
        last_compression()"""
        c = self.c
        c["updates"] += 1
        c["fifo_refresh"] += before.fifo_length > 0
        ctx = core + before.fifo_length
        if ctx > cfg.fifo_len:
            period, overflow = cfg.spkcache_update_period, ctx - cfg.fifo_len
            pop = min(max(period, overflow), ctx)
            c["pop_overflow" if overflow > period else "pop_period" if pop == period else "pop_context"] += 1
            c["popped"] += pop
        c["silent"] += after.silence_frames - before.silence_frames
        if comp is not None:
            self.compression(cfg, comp)

    def compression(self, cfg, comp):
        c = self.c
        K, sil, L = cfg.spkcache_len, cfg.spkcache_sil_frames_per_spk, comp.frames
        strong_k, weak_k, _ = k_values(cfg)
        thr = F32(cfg.pred_score_threshold)
        c["compressions"] += 1
        self.sizes.add((L + sil) * S)
        P, raw, dis = comp.preds, comp.scores, comp.disabled
        neg = dis == -np.inf
        nonpos = (P > 0.5) & (raw <= 0)
        c["half_preds"] += int((P == 0.5).sum())
        c["at_clip_bound"] += int(((P == thr) | (P == F32(1) - thr)).sum())
        c["zero_scores"] += int(((raw == 0) & (P > 0.5)).sum())
        c["nonpos_disabled"] += int((nonpos & neg).sum())
        c["nonpos_kept"] += int((nonpos & ~neg).sum())
        c["disabled_scores"] += int(neg.sum())
        c["latest_scored"] += int((~neg[K:]).sum())
        for stage, a, b, k in (("strong", dis, comp.strong, strong_k), ("weak", comp.strong, comp.weak, weak_k)):
            boosted = a != b
            if not boosted.any():
                c[f"{stage}_none"] += 1
            for spk in range(S):
                v = a[:, spk]
                finite = np.flatnonzero(v != -np.inf)
                nb = int(boosted[:, spk].sum())
                if k > 0 and len(finite) and nb == len(finite):
                    c[f"{stage}_all"] += 1
                elif nb:
                    c[f"{stage}_some"] += 1
                if 0 < k < len(finite):
                    order = finite[np.lexsort((finite, -v[finite]))]
                    c[f"ties_{stage}"] += int((v[order[k:]] == v[order[k - 1]]).sum())
        # the global selection over permuted = spk * (L + sil) + frame, the placeholders +inf
        F = L + sil
        perm = np.concatenate([np.concatenate([comp.weak[:, spk], np.full(sil, np.inf, np.float32)]) for spk in range(S)])
        order = np.lexsort((np.arange(perm.size), -perm.astype(np.float64)))
        kept, dropped = order[:K], order[K:]
        c["ties_topk"] += int((perm[dropped] == perm[kept[-1]]).sum())
        c["kept_neg_inf"] += int((perm[kept] == -np.inf).sum())
        c["disabled_slots"] += int(comp.is_disabled.sum())
        # recent frames (>= spkcacheLen) kept over older finite ones with a higher pre-boost score, or dropped under
        # them, by more than the two top-k boosts together could explain
        frame = np.where(np.arange(perm.size) % F < L, np.arange(perm.size) % F, -1)
        spk = np.arange(perm.size) // F
        pre = np.full(perm.size, -np.inf)
        real = frame >= 0
        pre[real] = np.where(neg[frame[real], spk[real]], -np.inf, raw[frame[real], spk[real]])
        recent = real & (frame >= K)
        old = real & (frame < K)
        is_kept = np.zeros(perm.size, bool)
        is_kept[kept] = True
        fin = np.isfinite(pre)
        margin = ((2 if strong_k > 0 else 0) + (1 if weak_k > 0 else 0)) * LN2 + 1e-3

        def beats(a, b):   # some a-element kept although a finite b-element dropped had a higher pre score by > 3 ln 2
            ka, db = pre[a & is_kept & fin], pre[b & ~is_kept & fin]
            return len(ka) and len(db) and db.max() > ka.min() + margin

        c["latest_reorder"] += bool(beats(recent, old) or beats(old, recent))

    def line(self, label):
        keys = ("compressions", "ties_strong", "ties_weak", "ties_topk", "kept_neg_inf", "disabled_slots",
                "zero_scores", "half_preds", "pop_period", "pop_overflow", "pop_context")
        return f"{label}: " + ", ".join(f"{k}={self.c[k]}" for k in keys) + f", N={sorted(self.sizes)}"


# ---- device handle against the oracle --------------------------------------------------------------------------------
def same_state(a, b):
    assert (a.spkcache_length, a.fifo_length, a.has_spkcache_preds, a.has_fifo_preds, a.silence_frames, a.chunks) == \
        (b.spkcache_length, b.fifo_length, b.has_spkcache_preds, b.has_fifo_preds, b.silence_frames, b.chunks)
    for k in ("spkcache", "fifo", "mean_silence"):
        assert np.array_equal(bits(getattr(a, k)), bits(getattr(b, k))), k
    for k in ("spkcache_preds", "fifo_preds"):
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None) == (y is None), k
        if x is not None:
            assert np.array_equal(bits(x), bits(y)), k


class Harness:
    """A SortformerStreams handle and one oracle session per open device session.  ``push`` draws each named
    session's model output, runs the oracle and the device (host or device variant), and checks the confirmed and
    tentative rows, the model inputs and, unless ``states`` is False, the pushed sessions' full snapshots."""

    def __init__(self, O, cfg, seed, max_core=0):
        self.O, self.cfg = O, cfg
        self.h = SortformerStreams(cfg, max_core)
        self.rng = np.random.default_rng(seed)
        self.ref, self.mode = {}, {}
        self.long_chunks = False   # contexts as sortformer_cases.contexts draws them, chunks up to max_core
        self.cov = Coverage()
        self.compressions = collections.Counter()   # per session

    def open(self, mode):
        sid = self.h.open()
        assert sid not in self.ref
        self.ref[sid], self.mode[sid] = self.O.Session(vars(self.h.config)), mode
        return sid

    def close(self, sid):
        self.h.close(sid)
        del self.ref[sid], self.mode[sid]
        self.compressions.pop(sid, None)

    def contexts(self, sid, streaming_rule):
        c, ref = self.h.config, self.ref[sid]
        if self.long_chunks:
            return contexts(self.rng, c, self.h.max_core, ref.chunks, not streaming_rule)
        lc = c.chunk_left_context if ref.chunks > 0 else 0
        core, rc = c.chunk_len, c.chunk_right_context
        if self.mode[sid] == "offline" and not streaming_rule and self.rng.random() < 0.3:   # a short (last) chunk
            core, rc = int(self.rng.integers(1, c.chunk_len + 1)), int(self.rng.integers(0, c.chunk_right_context + 1))
        return core, lc, rc

    def push(self, ids, device, streaming_rule, states=True):
        batch, outs = [], []
        for sid in ids:
            core, lc, rc = self.contexts(sid, streaming_rule)
            n = self.ref[sid].lengths()
            gen = "turns" if self.mode[sid] == "offline" else self.mode[sid]
            emb, preds = chunk(self.rng, gen, self.h.config, n.spkcache_length, n.fifo_length, core, lc, rc)
            batch.append((emb, preds, lc, rc))
        er = max(b[0].shape[0] for b in batch)
        pr = max(b[1].shape[0] for b in batch)
        E = np.full((len(ids), er, D), np.nan, np.float32)   # rows past a session's own are never read
        P = np.full((len(ids), pr, S), np.nan, np.float32)
        for i, (emb, preds, _, _) in enumerate(batch):
            E[i, :emb.shape[0]], P[i, :preds.shape[0]] = emb, preds
        el = np.array([b[0].shape[0] for b in batch], np.int32)
        lcs = None if streaming_rule else np.array([b[2] for b in batch], np.int32)
        rcs = None if streaming_rule else np.array([b[3] for b in batch], np.int32)
        for sid, (emb, preds, lc, rc) in zip(ids, batch):
            before = self.ref[sid].lengths()
            st, conf, tent = self.ref[sid].update(emb, preds, lc, rc)
            assert st == 0
            outs.append((conf, tent))
            comp = self.ref[sid].last_compression()
            self.cov.update(self.h.config, before, self.ref[sid].lengths(), conf.shape[0], comp)
            self.compressions[sid] += comp is not None
        if device:
            bufs = [_lib.DeviceBuffer(a.nbytes) for a in (E, P)]
            for b, a in zip(bufs, (E, P)):
                b.upload(a)
            dc, dt = _lib.DeviceBuffer(4 * len(ids) * er * S), _lib.DeviceBuffer(4 * len(ids) * er * S)
            cr, tr = self.h.update_device(ids, bufs[0], er, bufs[1], pr, dc, dt, el, lcs, rcs)
            _lib.synchronize()
            call = dc.download(len(ids) * er * S, np.float32)
            tall = dt.download(len(ids) * er * S, np.float32)
            conf = SortformerStreams._split(call, cr)
            tent = SortformerStreams._split(tall, tr)
            for b in bufs + [dc, dt]:
                b.free()
        else:
            conf, tent = self.h.update(ids, E, P, el, lcs, rcs)
        for (rc_, rt), c, t in zip(outs, conf, tent):
            assert np.array_equal(bits(c), bits(rc_)) and np.array_equal(bits(t), bits(rt))
        self.check_inputs(ids, device)
        if states:
            for sid in ids:
                same_state(self.h.state(sid), self.ref[sid].state())

    def check_inputs(self, ids, device):
        c = self.h.config
        if device:
            dsc, dff = _lib.DeviceBuffer(4 * len(ids) * c.spkcache_len * D), _lib.DeviceBuffer(4 * len(ids) * max(c.fifo_len, 1) * D)
            sl, fl = self.h.model_inputs_device(ids, dsc, dff)
            _lib.synchronize()
            sc = dsc.download((len(ids), c.spkcache_len, D), np.float32)
            ff = dff.download((len(ids), c.fifo_len, D), np.float32)
            dsc.free()
            dff.free()
        else:
            sc, ff, sl, fl = self.h.model_inputs(ids)
        for i, sid in enumerate(ids):
            rsc, rff, rsl, rfl = self.ref[sid].model_inputs()
            assert (sl[i], fl[i]) == (rsl, rfl)
            assert np.array_equal(bits(sc[i]), bits(rsc)) and np.array_equal(bits(ff[i]), bits(rff))
