"""Diarizer timelines on the H100 against the oracle (``oracle/oracle_timeline.cpp``), bit for bit.

Sessions run 1, 7 and 64 at a time under several configurations (sortformerDefault; pads and minimum durations; 7
speakers with logits; 32 speakers with maxStoredFrames 0).  Pushes name varying subsets in varying orders, carry empty
and tentative-only rows, predictions at the thresholds and NaN; sessions finalize mid-stream, clear a speaker, close and
reopen with the lowest free id, and the host and device variants alternate.  After every push both segment lists (order,
frames, activity bits), the per-session counts and the pushed sessions' full snapshots equal the oracle's.  Also: the
chain from Sortformer's device update, the offline case (64 one-hour files in one push), invalid arguments, and the
launch counts of a push and of finalize.
"""
import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.diarizer_timeline import SEGMENT, DiarizerTimelineConfig, DiarizerTimelines

F = np.float32


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_timeline
    oracle_timeline.build()
    oracle_timeline.lib()
    return oracle_timeline


CONFIGS = {
    "sortformer": DiarizerTimelineConfig.sortformer_default,
    "merge": lambda: DiarizerTimelineConfig(num_speakers=4, onset_pad_frames=2, offset_pad_frames=2, min_frames_on=4,
                                            min_frames_off=3, max_stored_frames=50),
    "logits7": lambda: DiarizerTimelineConfig(num_speakers=7, onset_threshold=0.6, offset_threshold=0.4,
                                              onset_pad_frames=1, min_frames_off=1, activity_type=1,
                                              max_stored_frames=13),
    "wide32": lambda: DiarizerTimelineConfig(num_speakers=32, offset_pad_frames=1, min_frames_on=1,
                                             max_stored_frames=0),
}


def draw(rng, rows, S):
    kind = rng.integers(0, 3)
    if kind == 0:
        return rng.choice(np.array([0.0, 0.25, 0.5, 0.75, 1.0, np.nan], F), size=(rows, S))
    if kind == 1:
        on = (rng.uniform(size=(rows // 5 + 1, S)) < 0.4).repeat(5, 0)[:rows]
        return np.where(on, rng.uniform(0.45, 1.0, (rows, S)), rng.uniform(0.0, 0.55, (rows, S))).astype(F)
    return rng.uniform(size=(rows, S)).astype(F)


def same_state(got, ref):
    assert got.finalized_frames == ref.finalized_frames
    assert got.stored.tobytes() == ref.stored.tobytes()
    assert got.tentative.tobytes() == ref.tentative.tobytes()
    assert got.scratch.tobytes() == ref.scratch.tobytes()


class Harness:
    def __init__(self, O, cfg, seed, max_tentative=12):
        self.O, self.cfg = O, cfg
        self.h = DiarizerTimelines(cfg, max_tentative)
        self.S, self.max_t = cfg.num_speakers, max_tentative
        self.rng = np.random.default_rng(seed)
        self.ref = {}

    def oracle_cfg(self):
        return {k: getattr(self.cfg, k) for k in ("num_speakers", "frame_duration_seconds", "onset_threshold",
                                                  "offset_threshold", "onset_pad_frames", "offset_pad_frames",
                                                  "min_frames_on", "min_frames_off", "activity_type",
                                                  "max_stored_frames")}

    def open(self):
        sid = self.h.open_session()
        assert sid not in self.ref
        self.ref[sid] = self.O.Timeline(self.oracle_cfg())
        return sid

    def close(self, sid):
        self.h.close(sid)
        del self.ref[sid]

    def push(self, ids, device):
        fin, ten = [], []
        for _ in ids:
            shape = self.rng.integers(0, 6)
            n = 0 if shape == 0 else int(self.rng.integers(1, 30))
            m = 0 if shape == 1 else int(self.rng.integers(0, self.max_t + 1))
            fin.append(draw(self.rng, n, self.S))
            ten.append(draw(self.rng, m, self.S))
        want = [self.ref[s].add_chunk(f, t) for s, f, t in zip(ids, fin, ten)]
        fr, tr = [a.shape[0] for a in fin], [a.shape[0] for a in ten]
        if device:
            fs, fc, ts, tc = push_device(self.h, ids, np.concatenate(fin), fr, np.concatenate(ten), tr)
        else:
            fs, fc, ts, tc = self.h.push_packed(ids, np.concatenate(fin), fr, np.concatenate(ten), tr)
        assert fc.tolist() == [len(w[0]) for w in want] and tc.tolist() == [len(w[1]) for w in want]
        assert fs.tobytes() == np.concatenate([w[0] for w in want]).tobytes()
        assert ts.tobytes() == np.concatenate([w[1] for w in want]).tobytes()
        for sid in ids:
            same_state(self.h.state(sid), self.ref[sid].state())


def push_device(h, ids, fin, fr, ten, tr):
    """push_device on freshly uploaded buffers; returns what push_packed returns"""
    bf, bt = h.segment_bound(fr, tr)
    bufs = [_lib.DeviceBuffer(max(a.nbytes, 4)) for a in (fin, ten)]
    for b, a in zip(bufs, (fin, ten)):
        if a.size:
            b.upload(a)
    dfs, dts = _lib.DeviceBuffer(SEGMENT.itemsize * bf), _lib.DeviceBuffer(SEGMENT.itemsize * bt)
    dfc, dtc = _lib.DeviceBuffer(8 * len(ids)), _lib.DeviceBuffer(8 * len(ids))
    h.push_device(ids, bufs[0], fr, bufs[1], tr, dfs, dts, dfc, dtc)
    _lib.synchronize()
    fc, tc = dfc.download(len(ids), np.int64), dtc.download(len(ids), np.int64)
    fs, ts = dfs.download(bf, SEGMENT)[:fc.sum()], dts.download(bt, SEGMENT)[:tc.sum()]
    for b in bufs + [dfs, dts, dfc, dtc]:
        b.free()
    return fs, fc, ts, tc


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("sessions", [1, 7, 64])
def test_sessions_match_the_oracle(gpu_lib, O, name, sessions):
    H = Harness(O, CONFIGS[name](), seed=sessions * 100 + len(name))
    for _ in range(sessions):
        H.open()
    for step in range(24):
        live = list(H.ref)
        k = max(1, int(len(live) * H.rng.uniform(0.5, 1.0)))
        ids = [int(s) for s in H.rng.permutation(live)[:k]]
        H.push(ids, device=step % 2 == 1)
        if step % 5 == 4:   # finalize a few sessions mid-stream
            fids = ids[:max(1, len(ids) // 2)]
            H.h.finalize(fids)
            for s in fids:
                H.ref[s].finalize()
                same_state(H.h.state(s), H.ref[s].state())
        if step % 7 == 6:   # removeSpeaker(clearCurrentSegment: true)
            s, spk = ids[0], int(H.rng.integers(0, H.S))
            H.h.clear_speaker(s, spk)
            H.ref[s].clear_speaker(spk)
            same_state(H.h.state(s), H.ref[s].state())
        if step % 9 == 8:
            s = ids[-1]
            H.h.reset([s])
            H.ref[s].reset()
            same_state(H.h.state(s), H.ref[s].state())
        if sessions > 1 and step % 6 == 5:   # close one and reopen the lowest free id
            s = min(H.ref)
            H.close(s)
            assert H.open() == s
    for sid in H.ref:
        same_state(H.h.state(sid), H.ref[sid].state())


@pytest.mark.gpu
def test_sortformer_device_update_chains_into_the_timeline(gpu_lib, O):
    from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams
    from oracle import oracle_sortformer as SF
    SF.build()
    D, S, n = 512, 4, 6
    sf = SortformerStreams(SortformerConfig.preset("default"))
    cfg = sf.config
    H = Harness(O, DiarizerTimelineConfig.sortformer_default(), seed=21, max_tentative=cfg.chunk_right_context)
    ids = [sf.open() for _ in range(n)]
    tl = [H.open() for _ in range(n)]
    refs = [SF.Session(vars(cfg)) for _ in range(n)]
    rng = np.random.default_rng(5)
    rows = cfg.chunk_left_context + cfg.chunk_len + cfg.chunk_right_context
    pred_rows = cfg.spkcache_len + cfg.fifo_len + rows
    dE, dP = _lib.DeviceBuffer(4 * n * rows * D), _lib.DeviceBuffer(4 * n * pred_rows * S)
    dc, dt = _lib.DeviceBuffer(4 * n * rows * S), _lib.DeviceBuffer(4 * n * rows * S)
    for step in range(50):
        lc = cfg.chunk_left_context if step else 0
        E = np.zeros((n, rows, D), F)
        P = np.full((n, pred_rows, S), np.nan, F)
        want = []
        for i in range(n):
            ln = refs[i].lengths()
            emb, preds = synth.sortformer_chunk(rng, "turns", ln.spkcache_length, ln.fifo_length, cfg.chunk_len, lc,
                                                cfg.chunk_right_context)
            E[i, :emb.shape[0]], P[i, :preds.shape[0]] = emb, preds
            _, conf, tent = refs[i].update(emb, preds, lc, cfg.chunk_right_context)
            want.append(H.ref[tl[i]].add_chunk(conf, tent))
        er = cfg.chunk_len + lc + cfg.chunk_right_context
        dE.upload(np.ascontiguousarray(E[:, :er]))
        dP.upload(P)
        cr, tr = sf.update_device(ids, dE, er, dP, pred_rows, dc, dt)
        _lib.synchronize()   # the Sortformer handle's stream wrote the rows
        bf, bt = H.h.segment_bound(cr, tr)
        dfs, dts = _lib.DeviceBuffer(SEGMENT.itemsize * bf), _lib.DeviceBuffer(SEGMENT.itemsize * bt)
        dfc, dtc = _lib.DeviceBuffer(8 * n), _lib.DeviceBuffer(8 * n)
        H.h.push_device(tl, dc, cr, dt, tr, dfs, dts, dfc, dtc)
        _lib.synchronize()
        fc, tc = dfc.download(n, np.int64), dtc.download(n, np.int64)
        assert dfs.download(bf, SEGMENT)[:fc.sum()].tobytes() == np.concatenate([w[0] for w in want]).tobytes()
        assert dts.download(bt, SEGMENT)[:tc.sum()].tobytes() == np.concatenate([w[1] for w in want]).tobytes()
        for b in (dfs, dts, dfc, dtc):
            b.free()
    for s in tl:
        same_state(H.h.state(s), H.ref[s].state())
    for b in (dE, dP, dc, dt):
        b.free()
    sf.close_handle()


@pytest.mark.gpu
def test_offline_hour_long_files_in_one_push(gpu_lib, O):
    """64 one-hour files [45 000 x 4] in one push, then finalize: rebuild(isComplete: true) of each"""
    files, T = 64, 45000
    cfg = DiarizerTimelineConfig.sortformer_default()
    cfg.max_stored_frames = T
    cfg.min_frames_off, cfg.offset_pad_frames = 2, 1
    H = Harness(O, cfg, seed=8, max_tentative=0)
    ids = [H.open() for _ in range(files)]
    rng = np.random.default_rng(9)
    preds = np.stack([draw(rng, T, 4) for _ in range(files)])
    fs, fc, ts, tc = H.h.push_packed(ids, preds, [T] * files, np.zeros((0, 4), F), [0] * files)
    H.h.finalize(ids)
    fo, to = 0, 0
    for i, s in enumerate(ids):
        # the tentative pass runs on no rows and still emits a held or trailing segment as tentative
        rf, rt = H.ref[s].rebuild(preds[i], is_complete=True)
        assert (fc[i], tc[i]) == (len(rf), len(rt))
        assert fs[fo:fo + fc[i]].tobytes() == rf.tobytes() and ts[to:to + tc[i]].tobytes() == rt.tobytes()
        fo, to = fo + fc[i], to + tc[i]
        same_state(H.h.state(s), H.ref[s].state())
    assert tc.sum() > 0


@pytest.mark.gpu
def test_invalid_arguments_leave_every_session_unchanged(gpu_lib, O):
    import ctypes as C
    H = Harness(O, CONFIGS["merge"](), seed=13, max_tentative=8)
    ids = [H.open() for _ in range(3)]
    closed = H.open()
    H.close(closed)
    for step in range(6):
        H.push(ids, device=step % 2 == 1)
    before = [H.h.state(s) for s in ids]
    L, S = gpu_lib, H.S

    def call(sessions, fr=(4, 4, 4), tr=(2, 2, 2), cap=None, count=None):
        sid = np.array(sessions, np.int32)
        m = sid.size if count is None else count
        fr, tr = np.array(fr[:m], np.int64), np.array(tr[:m], np.int64)
        f = np.full(max(1, int(fr.clip(0).sum()) * S), 0.9, F)
        t = np.full(max(1, int(tr.clip(0).sum()) * S), 0.9, F)
        out = np.zeros(10000, SEGMENT)
        fc, tc = np.zeros(max(m, 1), np.int64), np.zeros(max(m, 1), np.int64)
        return L.fa_diarizer_timeline_push(H.h._h, m, sid.ctypes.data, f.ctypes.data, fr.ctypes.data, t.ctypes.data,
                                           tr.ctypes.data, out.ctypes.data, out.size if cap is None else cap,
                                           out.ctypes.data, out.size, fc.ctypes.data, tc.ctypes.data)

    cases = {
        "duplicate": call([ids[0], ids[1], ids[0]]),
        "closed": call([ids[0], closed, ids[1]]),
        "too many tentative rows": call(ids, tr=(2, 9, 2)),
        "negative rows": call(ids, fr=(4, -1, 4)),
        "finalized output below the bound": call(ids, cap=3 * S * 3 - 1),
        "finalize closed": L.fa_diarizer_timeline_finalize(H.h._h, 1, np.array([closed], np.int32).ctypes.data),
        "reset duplicate": L.fa_diarizer_timeline_reset(H.h._h, 2, np.array([ids[0], ids[0]], np.int32).ctypes.data),
        "clear speaker out of range": L.fa_diarizer_timeline_clear_speaker(H.h._h, ids[0], S),
        "state of a closed session": L.fa_diarizer_timeline_session_state(H.h._h, closed,
                                                                          C.byref(_lib.TimelineSessionInfo()), None,
                                                                          None, None),
    }
    assert all(v == 1 for v in cases.values()), cases
    for s, b in zip(ids, before):
        same_state(H.h.state(s), b)
    H.push(ids, device=False)   # and the sessions go on as the oracle does


def _launches(fn):
    before = _lib.kernel_launch_count()
    fn()
    _lib.synchronize()
    return _lib.kernel_launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("sessions", [1, 64])
def test_launch_counts(gpu_lib, O, sessions):
    H = Harness(O, DiarizerTimelineConfig.sortformer_default(), seed=3, max_tentative=7)
    ids = [H.open() for _ in range(sessions)]
    rng = np.random.default_rng(2)
    fin, ten = rng.uniform(size=(sessions * 6, 4)).astype(F), rng.uniform(size=(sessions * 7, 4)).astype(F)
    assert _launches(lambda: H.h.push_packed(ids, fin, [6] * sessions, ten, [7] * sessions)) == 2
    assert _launches(lambda: push_device(H.h, ids, fin, [6] * sessions, ten, [7] * sessions)) == 2
    assert _launches(lambda: H.h.finalize(ids)) == 1                 # every session holds tentative rows
    assert _launches(lambda: H.h.finalize(ids)) == 0                 # none does now
    assert _launches(lambda: H.h.push_packed(ids, fin, [6] * sessions, ten[:0], [0] * sessions)) == 2
    assert _launches(lambda: H.h.finalize(ids)) == 0
    assert _launches(lambda: H.h.push_packed([], fin[:0], [], ten[:0], [])) == 0
    assert _launches(lambda: (H.h.reset(ids), H.h.clear_speaker(ids[0], 1))) == 0   # memsets
