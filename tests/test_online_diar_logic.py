"""Streaming speaker tracking on the CPU: the oracle (oracle/oracle_online_diar.cpp) on scenarios restated from the
reference's SpeakerManager and DiarizerManager behaviour, and the host build of online_diar_core.cuh
(tests/emul/online_diar_emul.cpp) held to the oracle bit for bit on seeded multi-chunk sessions."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle_online_diar as O

D = 256
R = O.resolved()


def unit(rng, n=1):
    x = rng.normal(size=(n, D)).astype(np.float32)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def logits_for(pattern):
    """[F x 7] logits whose argmax is pattern[f] (a powerset class)"""
    F = len(pattern)
    lg = np.zeros((F, 7), np.float32)
    lg[np.arange(F), pattern] = 5.0
    return lg


def speaker_rows(n, **kw):
    sp = np.zeros(n, O.SPEAKER)
    for k, v in kw.items():
        sp[k] = v
    return sp


def test_new_then_existing_speaker_and_fifo():
    rng = np.random.default_rng(1)
    s = O.Session()
    e = unit(rng)[0] * 3
    pattern = [1] * 300 + [0] * 289   # local speaker 0 alone for 300 frames
    embs = np.zeros((3, D), np.float32)
    embs[0] = e
    _, need, assigned, ids, vals = s.chunk(logits_for(pattern), 160000, embs, 0.0, R)
    assert list(need) == [1, 0, 0] and tuple(assigned[0]) == (0, 1) and len(ids) == 1
    assert vals[0, 0] == 0.0 and vals[0, 1] == np.float32(300 * 0.016875)
    for k in range(60):   # the same voice again: updates, and the FIFO stops at 50
        s.chunk(logits_for(pattern), 160000, embs, 10.0 * (k + 1), R)
    sp, cur, raws = s.read()
    assert len(sp) == 1 and sp[0]["raw_count"] == 50 and sp[0]["update_count"] == 61
    assert abs(float(np.linalg.norm(cur[0])) - 1) < 1e-5


def test_short_segment_does_not_create_a_speaker():
    s = O.Session()
    embs = np.zeros((3, D), np.float32)
    embs[0] = unit(np.random.default_rng(2))[0]
    # 50 frames: 0.84375 s < minSpeechDuration 1.0: no speaker, no segment
    _, _, assigned, ids, _ = s.chunk(logits_for([1] * 50 + [0] * 539), 160000, embs, 0.0, R)
    assert tuple(assigned[0]) == (-1, 0) and len(ids) == 0 and s.count() == (0, 1)


def test_activity_gate_is_strict_and_mask_gate_is_not():
    s = O.Session()
    embs = np.zeros((3, D), np.float32)
    embs[0] = unit(np.random.default_rng(3))[0]
    r = O.resolved(min_speech_duration=0.0)
    # exactly 10 active frames: the mask sum 10 is not < 10 (the model runs) but activity 10 is not > 10 (no id)
    _, need, assigned, _, _ = s.chunk(logits_for([1] * 10 + [0] * 579), 160000, embs, 0.0, r)
    assert need[0] == 1 and assigned[0, 0] == -1
    _, need, assigned, _, _ = s.chunk(logits_for([1] * 11 + [0] * 578), 160000, embs, 0.0, r)
    assert need[0] == 1 and assigned[0, 0] == 0


def test_powerset_ties_and_nan_take_the_first_index():
    s = O.Session()
    lg = np.zeros((589, 7), np.float32)
    lg[:, 2] = 1.0
    lg[:, 4] = 1.0          # tie between class 2 and class 4: class 2 (speaker 1 alone)
    lg[:100, 0] = np.nan    # NaN at index 0: index 0 stays (no speaker)
    lg[100:200, 1] = np.nan   # NaN past index 0 is never chosen
    masks, need, _, _, _ = s.chunk(lg, 160000, np.zeros((3, D), np.float32), 0.0, R)
    assert masks[1, :100].sum() == 0 and masks[1, 100:].sum() == 489 and masks[0].sum() == 0


def test_next_speaker_id_reset_overwrites_an_existing_speaker():
    rng = np.random.default_rng(4)
    s = O.Session()
    known = unit(rng, 3)
    sp = speaker_rows(3, key=[5, 1, 7], numeric=[5, 1, 7], has_numeric=1, update_count=1)
    s.initialize(sp[:2], known[:2], np.zeros((0, D), np.float32), mode=3)
    assert s.count() == (2, 6)
    s.initialize(speaker_rows(1, key=0, named=1, update_count=1), known[2:], np.zeros((0, D)), 3)
    assert s.count() == (3, 1)   # nextSpeakerId = the batch's largest numeric id (none) + 1
    embs = np.zeros((3, D), np.float32)
    embs[0] = -known[1] * 2      # far from everyone: a new speaker "1" replaces the known "1" in place
    _, _, assigned, _, _ = s.chunk(logits_for([1] * 300 + [0] * 289), 160000, embs, 0.0, R)
    sp_now, cur, _ = s.read()
    assert tuple(assigned[0]) == (0, 1) and len(sp_now) == 3 and sp_now[1]["key"] == 1
    assert s.count()[1] == 2 and not np.array_equal(cur[1], known[1])


def test_known_speaker_modes_and_permanence():
    rng = np.random.default_rng(5)
    s = O.Session()
    e = unit(rng, 4)
    sp = speaker_rows(2, key=[1, 2], numeric=[1, 2], has_numeric=1, update_count=1, permanent=[1, 0])
    s.initialize(sp, e[:2], np.zeros((0, D)), mode=3)
    new = speaker_rows(2, key=[1, 2], numeric=[1, 2], has_numeric=1, update_count=1)
    s.initialize(new, e[2:], np.zeros((0, D)), mode=2, preserve=True)   # overwrite: the permanent 1 stays
    _, cur, _ = s.read()
    assert np.dot(cur[0], e[0]) > 0.999 and np.dot(cur[1], e[3]) > 0.999   # 1 kept, 2 overwritten
    s.initialize(new[:1], e[3:], np.zeros((0, D)), mode=2, preserve=False)
    assert s.read()[0][0]["permanent"] == 0
    s.set_permanent(0, 2, True)
    s.reset(keep=True)
    sp_now, _, _ = s.read()
    assert list(sp_now["key"]) == [2] and s.count() == (1, 3)


def test_merge_keeps_the_fifty_most_recent_raws():
    rng = np.random.default_rng(6)
    s = O.Session()
    raws = rng.normal(size=(70, D)).astype(np.float32)
    sp = speaker_rows(2, key=[1, 2], numeric=[1, 2], has_numeric=1, update_count=[2, 3], raw_count=[40, 30])
    s.initialize(sp, unit(rng, 2), raws, mode=3)
    assert s.merge((0, 2), (0, 1))
    sp_now, cur, rw = s.read()
    assert len(sp_now) == 1 and sp_now[0]["raw_count"] == 50 and sp_now[0]["update_count"] == 5
    order = [int(np.argmax(np.abs(raws @ r))) for r in rw[0]]
    assert order == list(range(69, 19, -1))   # newest first


# ---- the host build of online_diar_core.cuh against the oracle
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("od") / "libod_emul.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul", "online_diar_emul.cpp")])
    L = C.CDLL(out)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.od_emul_new.restype = vp
    L.od_emul_free.argtypes = [vp]
    L.od_emul_chunk.argtypes = [vp, vp, i32, i64, vp, C.c_double, vp, vp, vp, vp, vp, vp]
    L.od_emul_chunk.restype = i32
    L.od_emul_count.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.od_emul_read.argtypes = [vp, vp, vp, vp]
    return L


def emul_chunk(L, p, logits, chunk_size, emb, offset, r):
    F = len(logits)
    bound = 3 * ((F + 1) // 2)
    masks, need = np.empty((3, F), np.float32), np.empty(3, np.int32)
    assigned = np.empty((3, 2), np.int64)
    ids, vals = np.empty((bound, 2), np.int64), np.empty((bound, 3), np.float32)
    n = L.od_emul_chunk(p, np.ascontiguousarray(logits, np.float32).ctypes.data, F, chunk_size,
                        np.ascontiguousarray(emb, np.float32).ctypes.data, offset,
                        np.ascontiguousarray(r, np.float32).ctypes.data, masks.ctypes.data, need.ctypes.data,
                        assigned.ctypes.data, ids.ctypes.data, vals.ctypes.data)
    return masks, need, assigned, ids[:n], vals[:n]


def same_speakers(a, b):
    """fa_od_speaker arrays equal field by field (the struct's padding is not compared)"""
    return len(a) == len(b) and all(a[f].tobytes() == b[f].tobytes() for f in O.SPEAKER.names)


def emul_read(L, p):
    c, nx = C.c_int64(), C.c_int64()
    L.od_emul_count(p, C.byref(c), C.byref(nx))
    sp = np.zeros(c.value, O.SPEAKER)
    cur, raws = np.zeros((c.value, D), np.float32), np.zeros((c.value, 50, D), np.float32)
    if c.value:
        L.od_emul_read(p, sp.ctypes.data, cur.ctypes.data, raws.ctypes.data)
    return (c.value, nx.value), sp, cur, raws


def random_chunk(rng, F, voices):
    """logits with runs of powerset classes, and embeddings near the session's voices (or degenerate)"""
    classes = np.repeat(rng.integers(0, 7, size=F // 20 + 1), 20)[:F]
    lg = rng.normal(size=(F, 7)).astype(np.float32)
    lg[np.arange(F), classes] += 4
    emb = np.empty((3, D), np.float32)
    for s in range(3):
        kind = rng.integers(0, 10)
        if kind == 0:
            emb[s] = 0
        elif kind == 1:
            emb[s] = rng.normal(size=D)
            emb[s, rng.integers(0, D)] = np.nan
        elif kind == 2:
            emb[s] = voices[rng.integers(0, len(voices))]   # an exact copy: a tie between equal speakers
        else:
            emb[s] = (voices[rng.integers(0, len(voices))] + rng.normal(0, 0.4, D).astype(np.float32)) * 3
    return lg, emb


@pytest.mark.parametrize("seed,F,chunk", [(0, 589, 160000), (1, 589, 80000), (2, 37, 160000), (3, 101, 320000)])
def test_core_host_build_equals_the_oracle(emul, seed, F, chunk):
    rng = np.random.default_rng(seed)
    voices = unit(rng, 6)
    r = O.resolved(min_speech_duration=0.3)
    ref, p = O.Session(), emul.od_emul_new()
    try:
        for k in range(40):
            lg, emb = random_chunk(rng, F, voices)
            want = ref.chunk(lg, chunk, emb, 10.0 * k, r)
            got = emul_chunk(emul, p, lg, chunk, emb, 10.0 * k, r)
            for g, w in zip(got, want):
                assert g.tobytes() == w.tobytes()
            (cnt, nx), sp, cur, raws = emul_read(emul, p)
            wsp, wcur, wraws = ref.read()
            assert (cnt, nx) == ref.count()
            assert same_speakers(sp, wsp) and cur.tobytes() == wcur.tobytes() and raws.tobytes() == wraws.tobytes()
        assert ref.count()[0] >= 3
    finally:
        emul.od_emul_free(p)


def test_thresholds_one_ulp_either_side(emul):
    """a query at distance exactly the threshold, and one ulp either side, against the strict < of assignSpeaker"""
    rng = np.random.default_rng(9)
    base = unit(rng)[0]
    for delta in (-1, 0, 1):
        ref, p = O.Session(), emul.od_emul_new()
        try:
            lg = logits_for([1] * 300 + [0] * 289)
            emb = np.zeros((3, D), np.float32)
            emb[0] = base
            ref.chunk(lg, 160000, emb, 0.0, R)
            emul_chunk(emul, p, lg, 160000, emb, 0.0, R)
            q = (base + rng.normal(0, 0.5, D)).astype(np.float32)
            d = ref.query(q)[0, 0]
            r = R.copy()
            r[0] = np.nextafter(d, np.float32(np.inf) if delta > 0 else -np.inf) if delta else d
            emb[0] = q
            want = ref.chunk(lg, 160000, emb, 10.0, r)
            got = emul_chunk(emul, p, lg, 160000, emb, 10.0, r)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
            assert (want[2][0, 1] == 1) == (delta > 0)
        finally:
            emul.od_emul_free(p)


def test_repeat_padding_for_five_second_chunks():
    audio = np.arange(1, 50001, dtype=np.float32)
    seg, wave = O.chunk_inputs(audio, 80000)
    assert np.array_equal(seg[:50000], audio) and not seg[50000:].any()
    padded = np.zeros(80000, np.float32)
    padded[:50000] = audio
    assert np.array_equal(wave, np.resize(padded, 160000))
    wave, mask = O.enrollment_inputs(audio[:1000], 589)
    assert np.array_equal(wave, np.resize(audio[:1000], 160000)) and mask.sum() == 589
    wave, mask = O.enrollment_inputs(audio[:100], 589)   # (589 * 100 + 80000) // 160000 == 0: a zero mask
    assert mask.sum() == 0
