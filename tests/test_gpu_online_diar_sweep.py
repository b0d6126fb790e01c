"""Streaming speaker tracking on the H100 against the oracle (oracle/oracle_online_diar.cpp), bit for bit: the model
inputs, the masks and need flags, the assigned ids, the segments and every session's whole database after every push,
for 1 to 4 096 sessions and random session subsets, with known speakers, merges, removals, permanence, resets and
queries interleaved, NaN / zero embeddings, host and device buffers, refused pushes that change nothing, and launch
counts."""
import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200 import online_diarizer as OD
from oracle import oracle_online_diar as O

pytestmark = pytest.mark.gpu

D = 256


def unit(rng, n):
    x = rng.normal(size=(n, D)).astype(np.float32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def random_chunk(rng, F, voices):
    classes = np.repeat(rng.integers(0, 7, size=F // 20 + 1), 20)[:F]
    lg = rng.normal(size=(F, 7)).astype(np.float32)
    lg[np.arange(F), classes] += 4
    if rng.integers(0, 8) == 0:
        lg[rng.integers(0, F), rng.integers(0, 7)] = np.nan
    emb = np.empty((3, D), np.float32)
    for s in range(3):
        kind = rng.integers(0, 13)
        if kind == 0:
            emb[s] = 0
        elif kind == 12:   # magnitude below validateEmbedding's 0.1
            emb[s] = unit(rng, 1)[0] * np.float32(rng.uniform(0.05, 0.1))
        elif kind == 1:
            emb[s] = rng.normal(size=D)
            emb[s, rng.integers(0, D)] = [np.nan, np.inf][int(rng.integers(0, 2))]
        elif kind == 2:
            emb[s] = voices[rng.integers(0, len(voices))]
        else:
            emb[s] = (voices[rng.integers(0, len(voices))] + rng.normal(0, 0.45, D).astype(np.float32)) * 3
    return lg, emb


def same_db(dbs, sid, ref):
    sp, cur, raws, nx = dbs.read_raw(sid)
    wsp, wcur, wraws = ref.read()
    assert (len(sp), nx) == ref.count()
    for f in O.SPEAKER.names:
        assert sp[f].tobytes() == wsp[f].tobytes(), f
    assert cur.tobytes() == wcur.tobytes() and raws.tobytes() == wraws.tobytes()


def push(dbs, sids, refs, rng, F, voices, tick, cfg, r, device=False):
    chunks = [rng.normal(size=int(rng.integers(0, 160001))).astype(np.float32) for _ in sids]
    seg, wave = OD.chunk_inputs(chunks, cfg)
    for j, c in enumerate(chunks):
        ws, ww = O.chunk_inputs(c, 160000)
        assert seg[j].tobytes() == ws.tobytes() and wave[j].tobytes() == ww.tobytes()
    data = [random_chunk(rng, F, voices) for _ in sids]
    lg = np.stack([d[0] for d in data])
    emb = np.stack([d[1] for d in data])
    offs = [10.0 * tick + 0.5 * j for j in range(len(sids))]
    if device:
        masks, need, assigned, counts, ids, vals = device_push(dbs, sids, lg, emb, offs, F)
    else:
        masks, need = dbs.embedding_inputs(sids, lg)
        assigned, counts, ids, vals = dbs.advance_raw(sids, emb, offs)
    for j, sid in enumerate(sids):
        wm, wn, wa, wi, wv = refs[sid].chunk(lg[j], 160000, emb[j], offs[j], r)
        assert masks[j].tobytes() == wm.tobytes() and need[j].tobytes() == wn.tobytes()
        assert assigned[j].tobytes() == wa.tobytes()
        assert counts[j] == len(wi) and ids[j, :counts[j]].tobytes() == wi.tobytes()
        assert vals[j, :counts[j]].tobytes() == wv.tobytes()


def device_push(dbs, sids, lg, emb, offs, F):
    import ctypes as C
    L = _lib.load()
    n = len(sids)
    bound = 3 * ((F + 1) // 2)
    s = np.ascontiguousarray(sids, np.int32)
    bufs = {k: _lib.DeviceBuffer(v) for k, v in dict(lg=lg.nbytes, masks=n * 3 * F * 4, need=n * 12, emb=emb.nbytes,
                                                    a=n * 48, c=n * 4, i=n * bound * 16, v=n * bound * 12).items()}
    bufs["lg"].upload(lg)
    bufs["emb"].upload(emb)
    cfg = dbs.config.c()
    _lib.check(L.fa_od_embedding_inputs_device(dbs._h, n, s.ctypes.data, bufs["lg"].ptr, C.byref(cfg),
                                               bufs["masks"].ptr, bufs["need"].ptr), "embedding_inputs_device")
    off = np.ascontiguousarray(offs, np.float64)
    _lib.check(L.fa_od_advance_device(dbs._h, n, s.ctypes.data, bufs["emb"].ptr, off.ctypes.data, C.byref(cfg),
                                      bufs["a"].ptr, bufs["c"].ptr, bufs["i"].ptr, bufs["v"].ptr), "advance_device")
    out = (bufs["masks"].download((n, 3, F), np.float32), bufs["need"].download((n, 3), np.int32),
           bufs["a"].download((n, 3, 2), np.int64), bufs["c"].download(n, np.int32),
           bufs["i"].download((n, bound, 2), np.int64), bufs["v"].download((n, bound, 3), np.float32))
    for b in bufs.values():
        b.free()
    return out


@pytest.mark.parametrize("sessions,ticks,F,device", [(1, 30, 589, False), (7, 12, 589, True), (64, 6, 101, False),
                                                       (4096, 2, 589, False)])
def test_pushes_equal_the_oracle(sessions, ticks, F, device):
    rng = np.random.default_rng(sessions)
    cfg = OD.DiarizerConfig(min_speech_duration=0.3)
    r = O.resolved(min_speech_duration=0.3)
    dbs = OD.SpeakerDatabases(F, cfg)
    sids = [dbs.open() for _ in range(sessions)]
    refs = {s: O.Session() for s in sids}
    voices = unit(rng, 8)
    before = _lib.kernel_launch_count()
    for t in range(ticks):
        pick = sids if t % 2 == 0 else sorted(rng.choice(sids, size=max(1, len(sids) // 2), replace=False).tolist())
        push(dbs, pick, refs, rng, F, voices, t, cfg, r, device)
    assert _lib.kernel_launch_count() - before == 3 * ticks
    for s in sids:
        same_db(dbs, s, refs[s])
    dbs.close_handle()


def test_database_operations_equal_the_oracle():
    rng = np.random.default_rng(11)
    cfg = OD.DiarizerConfig(min_speech_duration=0.3)
    r = O.resolved(min_speech_duration=0.3)
    F = 589
    dbs = OD.SpeakerDatabases(F, cfg)
    sids = [dbs.open() for _ in range(3)]
    refs = {s: O.Session() for s in sids}
    voices = unit(rng, 8)
    for t in range(40):
        push(dbs, sids, refs, rng, F, voices, t, cfg, r)
        sid = sids[t % 3]
        ref = refs[sid]
        op = t % 6
        if op == 0:   # known speakers in every mode
            n = int(rng.integers(1, 4))
            keys = rng.choice([1, 2, 3, 9, 40], size=n, replace=False)
            sp = np.zeros(n, O.SPEAKER)
            sp["key"] = sp["numeric"] = keys
            sp["has_numeric"] = 1
            sp["update_count"] = 1
            sp["duration"] = 2.5
            sp["permanent"] = rng.integers(0, 2, size=n)
            sp["raw_count"] = rng.integers(0, 51, size=n)
            cur = voices[rng.integers(0, 8, size=n)]
            raws = rng.normal(size=(int(sp["raw_count"].sum()), D)).astype(np.float32)
            mode, preserve = int(rng.integers(0, 4)), bool(rng.integers(0, 2))
            if rng.integers(0, 2):   # upsertSpeaker of the first one instead
                up = OD.Speaker(str(int(keys[0])), cur[0] * 2, 1.25, 3, raws[:int(sp["raw_count"][0])],
                                bool(sp["permanent"][0]))
                dbs.upsert_speaker(sid, up)
                row = sp[:1].copy()
                row["duration"], row["update_count"] = 1.25, 3
                ref.upsert(row, cur[0] * 2, raws[:int(sp["raw_count"][0])])
                same_db(dbs, sid, ref)
                continue
            ref.initialize(sp, cur, raws, mode, preserve)
            import ctypes as C
            _lib.check(_lib.load().fa_od_initialize(dbs._h, sid, n, np.ascontiguousarray(sp).ctypes.data,
                                                    np.ascontiguousarray(cur).ctypes.data,
                                                    raws.ctypes.data if raws.size else None, mode, int(preserve)),
                       "fa_od_initialize")
        elif op == 1:
            sp, _, _ = ref.read()
            if len(sp) >= 2:
                a, b = (int(k) for k in sp["key"][:2])
                assert dbs.merge_speaker(sid, str(a), str(b), bool(t % 4)) == ref.merge((0, a), (0, b), bool(t % 4))
        elif op == 2:
            sp, _, _ = ref.read()
            if len(sp):
                k = int(sp["key"][-1])
                assert dbs.set_permanent(sid, str(k), True) == ref.set_permanent(0, k, True)
        elif op == 3:
            sp, _, _ = ref.read()
            if len(sp):
                k = int(sp["key"][0])
                assert dbs.remove_speaker(sid, str(k), bool(t % 2)) == ref.remove(0, k, bool(t % 2))
        elif op == 4:
            dbs.reset(sid, bool(t % 4))
            ref.reset(bool(t % 4))
        q = np.concatenate([voices[:3], rng.normal(size=(2, D)).astype(np.float32)])
        assert dbs.distances(sid, q).tobytes() == ref.query(q).tobytes()
        assert device_query(dbs, sid, q).tobytes() == ref.query(q).tobytes()
        wsp, wcur, _ = ref.read()
        if len(wsp):
            d = ref.query(wcur)
            want = []
            for i in range(len(wsp)):
                for j in range(i + 1, len(wsp)):
                    if (wsp["permanent"][i] and wsp["permanent"][j]) or not d[i, j] < r[0]:
                        continue
                    a, b = str(int(wsp["key"][i])), str(int(wsp["key"][j]))
                    want.append((b, a) if not wsp["permanent"][j] else (a, b))
            assert dbs.find_mergeable_pairs(sid) == want
        same_db(dbs, sid, ref)
    dbs.close_handle()


def test_refused_push_changes_nothing_and_inputs():
    rng = np.random.default_rng(12)
    dbs = OD.SpeakerDatabases(589)
    a, b = dbs.open(), dbs.open()
    ref = O.Session()
    voices = unit(rng, 4)
    push(dbs, [a], {a: ref}, rng, 589, voices, 0, dbs.config, O.resolved())
    before = dbs.read_raw(a)
    with pytest.raises(_lib.FluidAudioError):   # b staged nothing: the whole push is refused
        dbs.advance_raw([a, b], np.zeros((2, 3, D), np.float32), [0.0, 0.0])
    after = dbs.read_raw(a)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before[:3], after[:3]))
    clips = [rng.normal(size=n).astype(np.float32) for n in (0, 1, 100, 1000, 159999, 200000)]
    wave, mask = OD.enrollment_inputs(clips, 589)
    for j, c in enumerate(clips):
        ww, wm = O.enrollment_inputs(c, 589)
        assert wave[j].tobytes() == ww.tobytes() and mask[j].tobytes() == wm.tobytes()
    cfg5 = OD.DiarizerConfig(chunk_duration=5.0)
    chunks = [rng.normal(size=n).astype(np.float32) for n in (80000, 30000, 120000)]
    seg, wave = OD.chunk_inputs(chunks, cfg5)
    for j, c in enumerate(chunks):
        ws, ww = O.chunk_inputs(c, 80000)
        assert seg[j].tobytes() == ws.tobytes() and wave[j].tobytes() == ww.tobytes()
    dbs.close_handle()


def device_query(dbs, sid, q):
    n = dbs.read_raw(sid)[0].shape[0]
    dq, dd = _lib.DeviceBuffer(q.nbytes), _lib.DeviceBuffer(max(1, len(q) * n * 4))
    dq.upload(np.ascontiguousarray(q, np.float32))
    _lib.check(_lib.load().fa_od_query_device(dbs._h, sid, len(q), dq.ptr, dd.ptr), "fa_od_query_device")
    out = dd.download((len(q), n), np.float32) if n else np.zeros((len(q), 0), np.float32)
    dq.free()
    dd.free()
    return out


def test_device_model_inputs_equal_the_host_ones():
    rng = np.random.default_rng(13)
    clips = [rng.normal(size=n).astype(np.float32) for n in (0, 5, 80000, 160000, 200000)]
    audio, off = OD._offsets(clips)
    n = len(clips)
    L = _lib.load()
    da, ds, dw, dm = (_lib.DeviceBuffer(max(4, x)) for x in (audio.nbytes, n * 640000, n * 640000, n * 589 * 4))
    da.upload(audio)
    _lib.check(L.fa_od_chunk_inputs_device(da.ptr, off.ctypes.data, n, 160000, ds.ptr, dw.ptr), "chunk_inputs_device")
    seg, wave = OD.chunk_inputs(clips)
    assert ds.download((n, 160000), np.float32).tobytes() == seg.tobytes()
    assert dw.download((n, 160000), np.float32).tobytes() == wave.tobytes()
    _lib.check(L.fa_od_enrollment_inputs_device(da.ptr, off.ctypes.data, n, 589, dw.ptr, dm.ptr), "enroll_device")
    wave, mask = OD.enrollment_inputs(clips, 589)
    assert dw.download((n, 160000), np.float32).tobytes() == wave.tobytes()
    assert dm.download((n, 589), np.float32).tobytes() == mask.tobytes()
    for b in (da, ds, dw, dm):
        b.free()


def test_many_enrollment_clips_pass_the_grid_limit():
    clips = [np.full(3, float(i % 7), np.float32) for i in range(65537)]
    audio, off = OD._offsets(clips)
    L = _lib.load()
    dw, dm = _lib.DeviceBuffer(len(clips) * 640000), _lib.DeviceBuffer(len(clips) * 4 * 4)
    da = _lib.DeviceBuffer(audio.nbytes)
    da.upload(audio)
    _lib.check(L.fa_od_enrollment_inputs_device(da.ptr, off.ctypes.data, len(clips), 4, dw.ptr, dm.ptr), "enroll")
    for i in (0, 65534, 65535, 65536):
        ww, wm = O.enrollment_inputs(clips[i], 4)
        row = np.empty(160000, np.float32)
        _lib.check(L.fa_memcpy_d2h(row.ctypes.data, dw.ptr.value + i * 640000, 640000), "d2h")
        assert row.tobytes() == ww.tobytes()
    for b in (da, dw, dm):
        b.free()


def test_perform_complete_diarization_equals_the_oracle_with_the_same_fakes():
    rng = np.random.default_rng(14)
    F = 589
    voices = unit(rng, 3)

    def seg_model(x):
        w = np.abs(x[:, :F * 7].reshape(-1, F, 7)) * 0 + 0.1
        t = ((np.arange(F) // 60 + np.int64(abs(float(x[0, 1000])) * 10)) % 7)
        w[:, np.arange(F), t] = 4.0
        return w.astype(np.float32)

    def emb_model(wave, mask):
        k = int(np.round(float(mask[0].sum()) + abs(float(wave[0, 77])) * 3)) % 3
        return (voices[k] * 2 + np.float32(0.01) * wave[0, 1000:1256]).astype(np.float32)[None]

    cfg = OD.DiarizerConfig(min_speech_duration=0.5)
    audio = rng.normal(size=16000 * 47 + 321).astype(np.float32)
    got = OD.DiarizerManager(seg_model, emb_model, cfg).perform_complete_diarization(audio, start_time=2.0)
    ref, want = O.Session(), []
    r = O.resolved(min_speech_duration=0.5)
    for at in range(0, len(audio), 160000):
        seg, wave = O.chunk_inputs(audio[at:at + 160000], 160000)
        lg = seg_model(seg[None])[0]
        masks, need, _, _, _ = ref.chunk(lg, 160000, np.zeros((3, D), np.float32), 0.0, r)   # no state change
        emb = np.zeros((3, D), np.float32)
        for s in range(3):
            if need[s]:
                emb[s] = emb_model(wave[None], masks[s][None])[0]
        _, _, _, ids, vals = ref.chunk(lg, 160000, emb, at / 16000 + 2.0, r)
        want += [(str(int(i[1])), v[0], v[1], v[2]) for i, v in zip(ids, vals)]
    assert len(want) > 3
    assert [(g.speaker_id, np.float32(g.start_time_seconds), np.float32(g.end_time_seconds),
             np.float32(g.quality_score)) for g in got] == want
