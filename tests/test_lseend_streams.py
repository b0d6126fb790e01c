"""LS-EEND live feature streams on the CPU: the reference's own tests ported onto the oracle (``oracle/oracle_lseend.cpp``),
the oracle pinned to an independent restatement (``tests/lseend_restated.py``), and the library's planning arithmetic
(``fluidaudio_b200/csrc/lseend/lseend_plan.h``, compiled through ``tests/emul/lseend_plan_shim.cpp``) against the oracle.
The GPU side is ``tests/test_gpu_lseend_stream_sweep.py``."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from lseend_restated import Provider as Restated, Queue, derived, push_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fluidaudio_b200", "csrc")
F32 = np.float32

# LSEENDFeatureProviderTests.makeMetadata (Tests/FluidAudioTests/Diarizer/LS-EEND/LSEENDFeatureProvider.swift:163-182)
TOY = dict(sample_rate=16000, n_mels=6, hop_length=4, win_length=16, context_size=7, subsampling=8, chunk_size=4,
           conv_delay=1)
CONFIGS = {
    "toy": TOY,
    "toy_negative_right": dict(TOY, context_size=3),          # mel right context 3 + 1 - 8 = -4
    "toy_no_delay": dict(TOY, conv_delay=0, chunk_size=1),
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


def make_audio(n):
    """LSEENDFeatureProviderTests.makeAudio (:146-153), in float32 as Swift evaluates it"""
    i = np.arange(n, dtype=F32)
    return (np.sin(i * F32(0.013)).astype(F32) * F32(0.25) + np.sin(i * F32(0.031)).astype(F32) * F32(0.1)).astype(F32)


def minimum_samples(cfg):
    n_fft, _, _, chunk_samples, _ = derived(cfg)
    return chunk_samples + n_fft // 2 - cfg["hop_length"]


def oracle_mel(O, cfg):
    mc = O.lseend_config(n_mels=cfg["n_mels"], n_fft=derived(cfg)[0], hop_length=cfg["hop_length"],
                         win_length=cfg["win_length"], sample_rate=cfg["sample_rate"])

    def mel(s):
        flat, ml, _ = O.mel_flat_transposed(mc, s, 0.0, 1, None)
        return flat[:ml].reshape(-1, cfg["n_mels"])
    return mel


# ------------------------------------------------------------------------------------------------ reference tests, ported
def test_queue_requires_exact_minimum_elements_for_first_chunk():
    """LSEENDQueueTests.testStreamingChunkQueueRequiresExactMinimumElementsForFirstChunk"""
    q = Queue(8, 3, 2, 1)
    assert not q.has_chunk() and q.ready == 0
    q.append(np.ones(9, F32))
    assert not q.has_chunk() and q.ready == 0
    q.append([1])
    assert q.has_chunk() and q.ready == 1
    assert q.pop_next().tolist() == [0, 0, 0] + [1] * 10
    assert q.ready == 0


def test_pop_all_chunks_consumes_only_whole_chunks_and_preserves_trailing_context():
    """LSEENDQueueTests.testPopAllChunksConsumesOnlyWholeChunksAndPreservesTrailingContext"""
    q = Queue(4, 2, 1, 1)
    q.append(np.arange(1, 11, dtype=F32))
    assert q.pop_all().tolist() == [0, 0] + list(range(1, 10))
    assert q.ready == 0
    q.append([11, 12, 13])
    assert q.pop_next().tolist() == list(range(7, 14))


def test_feature_provider_requires_exact_minimum_audio_for_first_chunk(OL):
    """LSEENDFeatureProviderTests.testFeatureProviderRequiresExactMinimumAudioForFirstChunk, on the oracle"""
    p = OL.Provider(TOY)
    n = minimum_samples(TOY)
    p.enqueue_audio(make_audio(n - 1))
    assert p.ready_chunks == 0 and p.emit_next_chunk() is None
    p.enqueue_audio(make_audio(1))
    f, mask, warmup = p.emit_next_chunk()
    assert f.size == OL.sizes(TOY).mel_frames * TOY["n_mels"]
    assert warmup == TOY["conv_delay"]


def test_chunked_mel_matches_non_chunked_pipeline_exactly(OL, oracle):
    """LSEENDFeatureProviderTests.testChunkedMelMatchesNonChunkedPipelineExactly, on the oracle: the provider's chunks
    equal the reference test's one-shot construction (whole buffer, one log-mel, one running mean, one mel queue) bit for
    bit, where the reference test allows 1e-6."""
    audio = make_audio(minimum_samples(TOY) * 3 + 37)
    p = OL.Provider(TOY)
    p.enqueue_audio(audio)
    p.drain_right_context_with_silence()
    got = []
    while (c := p.emit_next_chunk()) is not None:
        got.append(c[0])
    n_fft, mel_frames, chunk_mels, chunk_samples, flush = derived(TOY)
    buf = np.concatenate([np.zeros(n_fft // 2, F32), audio, np.zeros(flush, F32)])
    over = max(0, buf.size - (n_fft - TOY["hop_length"]))
    buf = np.concatenate([buf, np.zeros((chunk_samples - over % chunk_samples) % chunk_samples, F32)])
    feats, _, _ = oracle.lseend_features(oracle_mel_cfg(oracle), buf, np.zeros(TOY["n_mels"], F32), 0)
    q = Queue(chunk_mels, TOY["context_size"], TOY["context_size"] + 1 - TOY["subsampling"], TOY["n_mels"])
    q.append(feats)
    want = []
    while (c := q.pop_next()) is not None:
        want.append(c.reshape(mel_frames, -1))
    assert len(got) == len(want) > 0
    for a, b in zip(got, want):
        assert a.tobytes() == b.tobytes()


def oracle_mel_cfg(O):
    return O.lseend_config(n_mels=TOY["n_mels"], n_fft=16, hop_length=TOY["hop_length"], win_length=TOY["win_length"],
                           sample_rate=TOY["sample_rate"])


# ------------------------------------------------------------------------------------------------ oracle vs restatement
def same_state(a, b):
    return (a.audio.tobytes() == b["audio"].tobytes() and a.mel.tobytes() == b["mel"].tobytes() and
            a.cmn_mean.tobytes() == b["cmn_mean"].tobytes() and a.cmn_count == b["cmn_count"] and
            a.decoder_mask_end == b["decoder_mask_end"])


@pytest.mark.parametrize("name", list(CONFIGS))
def test_oracle_equals_restatement(OL, oracle, name):
    """Seeded push sequences (empty pushes, pushes below one hop, pushes of many chunks, drains followed by more audio,
    snapshot then rollback, reset): every chunk, mask, warm-up count and the whole state bit for bit."""
    cfg = CONFIGS[name]
    _, _, _, chunk_samples, _ = derived(cfg)
    rng = np.random.default_rng(sum(map(ord, name)))
    o, r = OL.Provider(cfg), Restated(cfg, mel=oracle_mel(oracle, cfg))
    snap = None
    emitted = 0
    for step, (n, drain) in enumerate(push_sequence(rng, chunk_samples, cfg["hop_length"], 60)):
        x = rng.standard_normal(n).astype(F32) * F32(0.1)
        got, want = o.push(x, drain), r.push(x, drain)
        for a, b in zip(got, want):
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), (name, step)
        emitted += len(got[2])
        assert same_state(o.state(), r.state()), (name, step)
        if step == 20:
            o.take_snapshot()
            snap = r.take_snapshot()
        if step == 40:
            o.rollback()
            r.rollback(snap)
            assert same_state(o.state(), r.state())
        if step == 50:
            o.reset()
            r.reset()
            assert same_state(o.state(), r.state())
    assert emitted > 10


# ------------------------------------------------------------------------------------------------ planning arithmetic
@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("lseend_plan") / "liblseend_plan.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I", CSRC, "-I", os.path.join(CSRC, "lseend"),
                           "-o", out,
                           os.path.join(ROOT, "tests", "emul", "lseend_plan_shim.cpp")])
    L = C.CDLL(out)
    L.lp_last_error.restype = C.c_char_p
    L.lp_resolve.argtypes = [C.c_void_p, C.c_void_p]
    L.lp_step.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def cfg_array(cfg, precision=0):
    keys = ("sample_rate", "n_mels", "hop_length", "win_length", "context_size", "subsampling", "chunk_size",
            "conv_delay")
    return np.array([cfg[k] for k in keys] + [precision], np.int32)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_planning_matches_oracle(plan, OL, name):
    """The derived sizes, and every push's chunk count, masks, warm-up counts and carried lengths, as the library plans
    them before anything runs, equal the oracle's after the push."""
    cfg = CONFIGS[name]
    c = cfg_array(cfg)
    sizes = np.zeros(10, np.int32)
    assert plan.lp_resolve(c.ctypes.data, sizes.ctypes.data) == 0
    assert sizes.tolist() == list(vars(OL.sizes(cfg)).values())
    rng = np.random.default_rng(7 + len(name))
    o = OL.Provider(cfg)
    lengths = np.zeros(4, np.int64)
    out = np.zeros(5, np.int64)
    _, _, _, chunk_samples, _ = derived(cfg)
    for step, (n, drain) in enumerate(push_sequence(rng, chunk_samples, cfg["hop_length"], 80)):
        masks = np.zeros(64 * cfg["chunk_size"] + 1, F32)
        warm = np.zeros(65, np.int32)
        assert plan.lp_step(c.ctypes.data, int(step == 0), lengths.ctypes.data, n, int(drain), out.ctypes.data,
                            masks.ctypes.data, warm.ctypes.data) == 0
        f, m, w = o.push(np.zeros(n, F32), drain)
        k = len(w)
        assert out[4] == k, (name, step)
        assert masks[:k * cfg["chunk_size"]].tobytes() == m.reshape(-1).tobytes() and warm[:k].tolist() == w.tolist()
        st = o.state()
        assert lengths.tolist() == [st.audio.size, st.mel.shape[0], st.cmn_count, st.decoder_mask_end], (name, step)
        assert st.audio.size < sizes[9] and st.mel.shape[0] < sizes[1]


@pytest.mark.parametrize("bad", [dict(hop_length=0), dict(n_mels=0), dict(subsampling=0), dict(chunk_size=0),
                                 dict(context_size=-1), dict(conv_delay=-1), dict(hop_length=17),
                                 dict(win_length=1 << 25, hop_length=4)])
def test_resolve_refuses_bad_configs(plan, bad):
    c = cfg_array(dict(TOY, **bad))
    assert plan.lp_resolve(c.ctypes.data, np.zeros(10, np.int32).ctypes.data) == 1
    assert plan.lp_last_error().startswith(b"lseend stream config")
    c = cfg_array(TOY, precision=2)
    assert plan.lp_resolve(c.ctypes.data, np.zeros(10, np.int32).ctypes.data) == 1


def test_entry_points_reject_null_handle():
    """No device needed: a NULL handle is refused with error text, and resolve needs none."""
    from fluidaudio_b200 import _lib
    try:
        L = _lib.load()
    except _lib.FluidAudioError:
        pytest.skip("library not built")
    assert L.fa_lseend_stream_chunks(None, 0, 10, 0) == -1
    assert L.fa_lseend_stream_open(None, None) == 1
    assert L.fa_lseend_stream_push(None, 0, None, None, None, None, None, 0, None, 0, None, 0, None) == 1
    for name in ("fa_lseend_stream_snapshot", "fa_lseend_stream_rollback", "fa_lseend_stream_reset"):
        assert getattr(L, name)(None, 0, None) == 1
    from fluidaudio_b200.lseend import LSEENDStreamConfig
    s = LSEENDStreamConfig(**TOY).resolve()
    assert (s.n_fft, s.mel_frames, s.chunk_samples, s.flush_samples, s.mask_length) == (16, 39, 128, 68, 5)
