"""LS-EEND live feature streams on the H100 (``-m gpu``) across metadata and both transform precisions.

Each session of a handle is driven by seeded push sequences (empty pushes, pushes below one hop, pushes of many chunks,
drains followed by more audio, snapshots, rollbacks and resets) and checked after every push:

* features bit for bit against the reference's own buffer construction (``tests/lseend_restated.py``: the audio queue's
  popAllChunks slices, each through the library's ``fa_mel_lseend_features`` with the running mean carried, appended to
  the mel queue and popped chunk by chunk);
* masks, warm-up counts, chunk counts and the session's state (unread audio, cmnCount, decoderMaskEnd) exactly against
  the oracle (``oracle/oracle_lseend.cpp``), its unread mel rows and running mean bit for bit against the restatement;
* the whole chain of a session that is never rolled back within the LS-EEND bar of ``test_gpu_mel_adapter_sweep.py``
  against the oracle's own log-mel.

The toy metadata of the reference's tests has nFFT 16, below the mel kernels' 32: creating it is refused, and the sweep
runs its queue shape (6 mels, context 7, subsampling 8, chunk 4, conv delay 1) at win 32, hop 8 instead."""
import ctypes as C

import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200.lseend import LSEENDFeatureProvider, LSEENDFeatureStreams, LSEENDStreamConfig
from fluidaudio_b200.mel import Precision
from lseend_restated import Provider as Restated, derived, push_sequence
from test_gpu_mel_adapter_sweep import _bar_for, _bar_name, _kind_of, check_lseend_end_to_end, lseend, \
    lseend_handle, prepadded_mel

F32 = np.float32
INVALID_ARGUMENT, UNSUPPORTED = 1, 8
TOY = dict(sample_rate=16000, n_mels=6, hop_length=4, win_length=16, context_size=7, subsampling=8, chunk_size=4,
           conv_delay=1)
CONFIGS = {
    "toy32": dict(TOY, hop_length=8, win_length=32),
    "toy32_negative_right": dict(TOY, hop_length=8, win_length=32, context_size=3),
    "8k": dict(sample_rate=8000, n_mels=23, hop_length=80, win_length=200, context_size=7, subsampling=10,
               chunk_size=1, conv_delay=2),
    "16k": dict(sample_rate=16000, n_mels=23, hop_length=160, win_length=400, context_size=7, subsampling=10,
                chunk_size=2, conv_delay=2),
}


@pytest.fixture(scope="module")
def OL():
    from oracle import oracle_lseend
    oracle_lseend.build()
    oracle_lseend.lib()
    return oracle_lseend


def library_features(m):
    """processAudioQueue's log-mel, scaling and running mean of one slice through fa_mel_lseend_features on handle m."""
    return lambda s, mean, count: lseend(m, np.ascontiguousarray(s, F32), mean, count)


def same_bits(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def check_state(streams, sid, o, r, what):
    got, want = streams.state(sid), o.state()
    assert same_bits(got.audio, want.audio), what
    assert (got.cmn_count, got.decoder_mask_end) == (want.cmn_count, want.decoder_mask_end), what
    assert got.mel.shape == want.mel.shape, what
    rs = r.state()
    assert same_bits(got.mel, rs["mel"]) and same_bits(got.cmn_mean, rs["cmn_mean"]), what
    return got


@pytest.mark.gpu
def test_toy_metadata_below_kernel_limits_is_refused(gpu_lib):
    cfg = LSEENDStreamConfig(**TOY)
    assert cfg.resolve().n_fft == 16
    h = C.c_void_p()
    assert gpu_lib.fa_lseend_stream_create(C.byref(cfg._c()), C.byref(h)) == UNSUPPORTED and not h.value


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [Precision.f64, Precision.f32])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_streams_match_reference_construction(gpu_lib, oracle, OL, name, prec):
    cfg = CONFIGS[name]
    n_fft, _, _, chunk_samples, _ = derived(cfg)
    streams = LSEENDFeatureStreams(LSEENDStreamConfig(**cfg, precision=int(prec)))
    m, _ = lseend_handle(sample_rate=cfg["sample_rate"], n_mels=cfg["n_mels"], win_length=cfg["win_length"],
                         hop_length=cfg["hop_length"])
    m.set_precision(prec)
    S = 3
    ids = [streams.open() for _ in range(S)]
    orc = [OL.Provider(cfg) for _ in range(S)]
    res = [Restated(cfg, features=library_features(m)) for _ in range(S)]
    rng = np.random.default_rng(int(prec) * 100 + len(name))
    seqs = [push_sequence(rng, chunk_samples, cfg["hop_length"], 40) for _ in range(S)]
    snaps, snap_state = {}, {}
    emitted = 0
    for step in range(40):
        tick = [i for i in range(S) if rng.random() < 0.8]
        chunks = {ids[i]: (rng.standard_normal(seqs[i][step][0]) * 0.1).astype(F32) for i in tick}
        drain = [ids[i] for i in tick if seqs[i][step][1]]
        planned = {ids[i]: streams.chunks(ids[i], chunks[ids[i]].size, ids[i] in drain) for i in tick}
        before = _lib.kernel_launch_count()
        out = streams.push(chunks, drain)
        launches = _lib.kernel_launch_count() - before
        capacity = streams.sizes.audio_capacity
        completes = any(ids[i] in drain or orc[i].state().audio.size + chunks[ids[i]].size >= capacity for i in tick)
        receives = any(chunks[ids[i]].size for i in tick) or drain
        assert launches == (4 if completes else 1 if receives else 0), (name, step, launches)
        for i in tick:
            what = dict(config=name, precision=int(prec), step=step, session=i)
            f, mk, w = out[ids[i]]
            of, om, ow = orc[i].push(chunks[ids[i]], ids[i] in drain)
            rf, _, _ = res[i].push(chunks[ids[i]], ids[i] in drain)
            assert len(w) == len(ow) == planned[ids[i]], what
            assert same_bits(mk, om) and same_bits(w, ow), what
            assert same_bits(f, rf), what
            emitted += len(w)
            check_state(streams, ids[i], orc[i], res[i], what)
        # sessions 1 and 2 snapshot, roll back and reset; session 0 runs one chain from a fresh state
        if step == 12:
            streams.snapshot(ids[1:])
            for i in (1, 2):
                orc[i].take_snapshot()
                snaps[i] = res[i].take_snapshot()
                snap_state[i] = streams.state(ids[i])
        if step == 25:
            before = _lib.kernel_launch_count()
            streams.rollback(ids[1:])
            assert _lib.kernel_launch_count() - before == 1
            for i in (1, 2):
                orc[i].rollback()
                res[i].rollback(snaps[i])
                got = check_state(streams, ids[i], orc[i], res[i], (name, "rollback", i))
                want = snap_state[i]
                assert same_bits(got.audio, want.audio) and same_bits(got.mel, want.mel) and \
                    same_bits(got.cmn_mean, want.cmn_mean), (name, "rollback restores the snapshot")
        if step == 32:
            streams.reset([ids[2]])
            orc[2].reset()
            res[2].reset()
            got = check_state(streams, ids[2], orc[2], res[2], (name, "reset"))
            fresh = streams.open()
            want = streams.state(fresh)
            streams.close(fresh)
            assert same_bits(got.audio, want.audio) and same_bits(got.mel, want.mel) and \
                same_bits(got.cmn_mean, want.cmn_mean) and got.has_snapshot
    assert emitted > 20
    # session 0's whole chain against the oracle's own log-mel
    kind = _kind_of(m)
    ocfg = oracle.lseend_config(n_mels=cfg["n_mels"], n_fft=n_fft, hop_length=cfg["hop_length"],
                                win_length=cfg["win_length"], sample_rate=cfg["sample_rate"])
    slices = res[0].slices
    assert slices
    lib_rows, lib_mels, ref_rows, ref_mels = [], [], [], []
    lm, lc, rm, rc = np.zeros(cfg["n_mels"], F32), 0, np.zeros(cfg["n_mels"], F32), 0
    for s in slices:
        f, lm, lc = lseend(m, s, lm, lc)
        lib_rows.append(f)
        lib_mels.append(prepadded_mel(m, s))
        f, rm, rc = oracle.lseend_features(ocfg, s, rm, rc)
        ref_rows.append(f)
        ref_mels.append(oracle.mel_flat_transposed(ocfg, s, 0.0, 1, None)[0].reshape(-1, cfg["n_mels"]))
    check_lseend_end_to_end(np.concatenate(lib_rows), np.concatenate(lib_mels), np.concatenate(ref_rows),
                            np.concatenate(ref_mels), _bar_for(kind, prec), f"lseend stream {_bar_name(kind, prec)}",
                            dict(config=name, precision=int(prec)))
    m.close()
    streams.close_handle()


@pytest.mark.gpu
def test_failed_pushes_change_nothing(gpu_lib):
    cfg = CONFIGS["16k"]
    streams = LSEENDFeatureStreams(LSEENDStreamConfig(**cfg))
    a, b = streams.open(), streams.open()
    rng = np.random.default_rng(3)
    streams.push({a: rng.standard_normal(5000).astype(F32), b: rng.standard_normal(3000).astype(F32)})
    closed = streams.open()
    streams.close(closed)
    before = [streams.state(s) for s in (a, b)]
    x = rng.standard_normal(8000).astype(F32)
    L, h = gpu_lib, streams._h
    k = streams.chunks(a, x.size)
    assert k > 0
    F, T = streams.sizes.mel_frames * cfg["n_mels"], cfg["chunk_size"]
    feats, masks, warm = np.zeros(k * F, F32), np.zeros(k * T, F32), np.zeros(k, np.int32)
    counts = np.zeros(2, np.int64)

    def raw(ids, offsets, f_len=feats.size, m_len=masks.size, w_len=warm.size):
        ids = np.array(ids, np.int32)
        offsets = np.array(offsets, np.int64)
        return L.fa_lseend_stream_push(h, ids.size, ids.ctypes.data, x.ctypes.data, offsets.ctypes.data, None,
                                       feats.ctypes.data, f_len, masks.ctypes.data, m_len, warm.ctypes.data, w_len,
                                       counts.ctypes.data)

    launches = _lib.kernel_launch_count()
    assert raw([a, a], [0, 4000, 8000]) == INVALID_ARGUMENT            # duplicate session
    assert raw([a, closed], [0, 4000, 8000]) == INVALID_ARGUMENT       # closed session
    assert raw([a, b], [0, 5000, 4000]) == INVALID_ARGUMENT            # decreasing offsets
    assert raw([a], [0, 8000], f_len=feats.size - 1) == INVALID_ARGUMENT
    assert raw([a], [0, 8000], m_len=masks.size - 1) == INVALID_ARGUMENT
    assert raw([a], [0, 8000], w_len=k - 1) == INVALID_ARGUMENT
    assert L.fa_lseend_stream_rollback(h, 1, np.array([a], np.int32).ctypes.data) == INVALID_ARGUMENT   # no snapshot
    assert _lib.kernel_launch_count() == launches
    for s, want in zip((a, b), before):
        got = streams.state(s)
        assert same_bits(got.audio, want.audio) and same_bits(got.mel, want.mel) and \
            same_bits(got.cmn_mean, want.cmn_mean) and got.cmn_count == want.cmn_count
    assert raw([a], [0, 8000]) == 0 and counts[0] == k
    streams.close_handle()


@pytest.mark.gpu
@pytest.mark.parametrize("sessions", [1, 64, 700])
def test_launches_per_push_and_device_push(gpu_lib, sessions):
    """Four launches for a push in which some session completes an audio chunk, one when samples only join carries,
    none for an empty push, whatever the session count; push_device equals push bit for bit on a twin handle."""
    cfg = CONFIGS["16k"]
    host = LSEENDFeatureStreams(LSEENDStreamConfig(**cfg))
    dev = LSEENDFeatureStreams(LSEENDStreamConfig(**cfg))
    hid = [host.open() for _ in range(sessions)]
    did = [dev.open() for _ in range(sessions)]
    rng = np.random.default_rng(sessions)
    F, T = host.sizes.mel_frames * cfg["n_mels"], cfg["chunk_size"]
    cap = 64 * sessions
    d_feat, d_mask, d_warm = (_lib.DeviceBuffer(cap * F * 4), _lib.DeviceBuffer(cap * T * 4), _lib.DeviceBuffer(cap * 4))
    for tick, n in enumerate((100, 0, 1600, 1600, 17, 48000, 0)):
        drain = tick == 5
        xs = [(rng.standard_normal(n) * 0.1).astype(F32) for _ in range(sessions)]
        k = [host.chunks(s, n, drain) for s in hid]
        carry = host.state(hid[0]).audio.size
        before = _lib.kernel_launch_count()
        out = host.push(dict(zip(hid, xs)), hid if drain else ())
        launches = _lib.kernel_launch_count() - before
        completes = drain or carry + n >= host.sizes.audio_capacity
        assert launches == (4 if completes else (1 if n else 0)), (tick, launches)
        audio = np.concatenate(xs) if n else np.zeros(1, F32)
        d_audio = _lib.DeviceBuffer(audio.nbytes)
        d_audio.upload(audio)
        offsets = np.arange(sessions + 1, dtype=np.int64) * n
        counts = dev.push_device(did, d_audio, offsets, d_feat, d_mask, d_warm,
                                 drain=np.full(sessions, int(drain), np.int32))
        assert counts.tolist() == k
        total = int(sum(k))
        _lib.synchronize()
        if total:
            f = d_feat.download(total * F, F32).reshape(total, -1, cfg["n_mels"])
            mk = d_mask.download(total * T, F32).reshape(total, T)
            w = d_warm.download(total, np.int32)
            c = 0
            for s, kk in zip(hid, k):
                hf, hm, hw = out[s]
                assert same_bits(f[c:c + kk], hf) and same_bits(mk[c:c + kk], hm) and same_bits(w[c:c + kk], hw)
                c += kk
        d_audio.free()
    before = _lib.kernel_launch_count()
    host.snapshot(hid)
    host.rollback(hid)
    host.reset(hid)
    assert _lib.kernel_launch_count() - before == 3
    host.close_handle()
    dev.close_handle()


@pytest.mark.gpu
def test_provider_facade_follows_the_reference_class(gpu_lib, OL):
    """LSEENDFeatureProvider: the reference test's exact minimum (on the sweep's toy shape), emit_next_chunk one chunk at
    a time, and a snapshot that keeps the chunks not yet emitted."""
    cfg = CONFIGS["toy32"]
    n_fft, _, _, chunk_samples, _ = derived(cfg)
    p = LSEENDFeatureProvider(LSEENDStreamConfig(**cfg))
    o = OL.Provider(cfg)
    minimum = chunk_samples + n_fft // 2 - cfg["hop_length"]
    x = (np.sin(np.arange(10 * minimum, dtype=F32) * F32(0.013)) * F32(0.25)).astype(F32)
    p.enqueue_audio(x[:minimum - 1])
    o.enqueue_audio(x[:minimum - 1])
    assert p.ready_chunks == o.ready_chunks == 0 and p.emit_next_chunk() is None
    p.enqueue_audio(x[minimum - 1:minimum])
    f, mk, w = p.emit_next_chunk()
    assert w == cfg["conv_delay"] and f.shape == (o.mel_frames, cfg["n_mels"])
    p.enqueue_audio(x[minimum:])
    p.take_snapshot()
    ready = p.ready_chunks
    assert ready > 2
    first = p.emit_next_chunk()
    p.drain_right_context_with_silence()
    p.rollback()
    assert p.ready_chunks == ready
    again = p.emit_next_chunk()
    assert same_bits(again[0], first[0]) and same_bits(again[1], first[1]) and again[2] == first[2]
    p.reset()
    assert p.ready_chunks == 0 and p.streams.state(p.session).audio.size == n_fft // 2
