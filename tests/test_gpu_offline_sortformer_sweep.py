"""Offline Sortformer windows on the H100 against the oracle (oracle/oracle_offline_sortformer.cpp): model inputs for
1 … 4 096 files at the frame-count edges, one-hour files and every overlap edge; the stitch on the same inputs, on the
adversarial prediction sets, at overlap 383 (a frame averaged up to 384 times) and on a planted case whose mappings
must invert known permutations; host against device variants with one launch each; refusals that write nothing; and
process_complete_batch end to end against the oracle's processComplete fed the library's own mel rows."""
import numpy as np
import pytest

import offline_sortformer_cases as K
from fluidaudio_b200 import _lib
from fluidaudio_b200.diarizer_timeline import DiarizerTimelineConfig
from fluidaudio_b200.mel import AudioMelSpectrogram
from fluidaudio_b200.offline_sortformer import OfflineSortformerDiarizer, OfflineSortformerWindows
from oracle import oracle_offline_sortformer as O

pytestmark = pytest.mark.gpu

WINDOW = 128 * 3072


@pytest.fixture(scope="module", autouse=True)
def device():
    if _lib.device_count() < 1:
        pytest.skip("needs an H100")
    _lib.set_device(0)


@pytest.fixture(scope="module")
def win():
    return OfflineSortformerWindows()


def same_bits(a, b):
    """bit for bit, any NaN equal to any NaN (payloads are not compared)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and np.array_equal(np.where(both, 0, a).view(np.uint32),
                                                 np.where(both, 0, b).view(np.uint32))


def packed(rng, frames, gap=0):
    """the files' time-major rows packed with `gap` spare rows after each, and their float offsets"""
    rows = [K.mel_rows(rng, n) for n in frames]
    offsets, at = [], 0
    for r in rows:
        offsets.append(at)
        at += (r.shape[0] + gap) * 128
    mel = np.zeros(max(at, 1), np.float32)
    for r, o in zip(rows, offsets):
        mel[o:o + r.size] = r.reshape(-1)
    return mel, np.array(offsets, np.int64), rows


def check_model_inputs(got_mel, got_len, rows, frames, overlap, first=0):
    """the windows [first, first + len(got_len)) of the files against the oracle's copy"""
    k = 0
    for r, n in zip(rows, frames):
        nw = int(OfflineSortformerWindows().plan([n], overlap)[0][0])
        hop = (384 - max(0, min(overlap, 383))) * 8
        for j in range(nw):
            if first <= k < first + len(got_len):
                start = j * hop
                valid = min(3072, n - start)
                want, ml = O.run_offline(r[start:start + valid], valid)
                assert got_len[k - first] == ml and got_mel[k - first].tobytes() == want.tobytes(), (n, j, overlap)
            k += 1


@pytest.mark.parametrize("overlap", K.OVERLAP_EDGES)
def test_model_inputs_at_the_frame_edges(win, overlap):
    rng = np.random.default_rng(abs(overlap) % 1000 + 1)
    frames = list(K.FRAME_EDGES) + [0, 7777]
    mel, off, rows = packed(rng, frames, gap=5)
    got, ml = win.model_inputs(mel, off, frames, overlap)
    check_model_inputs(got, ml, rows, frames, overlap)


def test_model_inputs_for_many_files_and_an_hour(win):
    rng = np.random.default_rng(2)
    for frames in ([int(x) for x in rng.integers(1, 700, size=4096)], [K.HOUR, 3001, K.HOUR]):
        mel, off, rows = packed(rng, frames)
        w, _ = win.plan(frames, 100)
        W = int(w.sum())
        d_mel = _lib.DeviceBuffer(mel.nbytes)
        d_mel.upload(mel)
        d_out, d_len = _lib.DeviceBuffer(W * WINDOW * 4), _lib.DeviceBuffer(W * 4)
        before = _lib.kernel_launch_count()
        win.model_inputs_device(d_mel.ptr, off, frames, W, d_out.ptr, d_len.ptr, 100)
        _lib.synchronize()
        assert _lib.kernel_launch_count() - before == 1
        ml = d_len.download(W, np.int32)
        for first in range(0, W, 256):
            n = min(256, W - first)
            chunk = np.empty((n, 128, 3072), np.float32)
            _lib.check(_lib.load().fa_memcpy_d2h(chunk.ctypes.data, d_out.ptr.value + first * WINDOW * 4,
                                                 chunk.nbytes), "fa_memcpy_d2h")
            check_model_inputs(chunk, ml[first:first + n], rows, frames, 100, first)
        for b in (d_mel, d_out, d_len):
            b.free()


def oracle_stitch(frames, overlap, preds):
    """the oracle's loop per file, its k-th model call answered with the file's k-th window of preds"""
    w, _ = OfflineSortformerWindows().plan(frames, overlap)
    out, maps, at = [], [], 0
    for n, nw in zip(frames, w.tolist()):
        calls = iter(preds[at:at + nw])
        g, m = O.stitch(np.zeros((int(n), 128), np.float32), n, overlap, lambda mel, ml: next(calls))
        out.append(g)
        maps.append(m)
        at += nw
    return np.concatenate(out), np.concatenate(maps)


def check_stitch(win, frames, overlap, preds):
    got, maps = win.stitch(preds, frames, overlap, mappings=True)
    want, want_maps = oracle_stitch(frames, overlap, preds)
    assert same_bits(got, want) and np.array_equal(maps, want_maps), (frames, overlap)
    return got, maps


@pytest.mark.parametrize("overlap", K.OVERLAP_EDGES)
def test_stitch_at_the_frame_edges(win, overlap):
    rng = np.random.default_rng(abs(overlap) % 1000 + 5)
    frames = list(K.FRAME_EDGES) + [0, 7777, 12345]
    w, _ = win.plan(frames, overlap)
    check_stitch(win, frames, overlap, K.adversarial_preds(rng, int(w.sum()), "random"))


@pytest.mark.parametrize("kind", K.KINDS)
def test_stitch_on_adversarial_predictions(win, kind):
    rng = np.random.default_rng(len(kind) * 11)
    for overlap in (1, 2, 37, 100, 200, 382, 383):
        frames = [3073, 5344, 9000, 3072, 1]
        w, _ = win.plan(frames, overlap)
        check_stitch(win, frames, overlap, K.adversarial_preds(rng, int(w.sum()), kind))


def test_stitch_at_overlap_383_and_for_an_hour(win):
    rng = np.random.default_rng(9)
    frames = [9000, 3073]
    w, _ = win.plan(frames, 383)
    check_stitch(win, frames, 383, K.adversarial_preds(rng, int(w.sum()), "random"))
    frames = [K.HOUR, K.HOUR - 5000]
    w, _ = win.plan(frames, 100)
    check_stitch(win, frames, 100, K.adversarial_preds(rng, int(w.sum()), "random"))


@pytest.mark.parametrize("overlap", [20, 100, 383])
def test_stitch_inverts_planted_permutations(win, overlap):
    rng = np.random.default_rng(overlap)
    frames = 20000 if overlap < 383 else 4000
    preds, perms, truth = K.planted(rng, frames, overlap)
    got, maps = check_stitch(win, [frames], overlap, preds)
    for k in range(perms.shape[0]):
        assert maps[k].tolist() == np.argsort(perms[k]).tolist(), k
    assert np.abs(got - truth).max() < 1e-6


def test_host_and_device_variants_agree_with_one_launch_each(win):
    rng = np.random.default_rng(21)
    frames = [3001, 0, 5344, 3072, 20000]
    mel, off, _ = packed(rng, frames, gap=3)
    w, r = win.plan(frames, 100)
    W, R = int(w.sum()), int(r.sum())
    before = _lib.kernel_launch_count()
    host_mel, host_len = win.model_inputs(mel, off, frames, 100)
    assert _lib.kernel_launch_count() - before == 1
    d_mel, d_out, d_len = _lib.DeviceBuffer(mel.nbytes), _lib.DeviceBuffer(W * WINDOW * 4), _lib.DeviceBuffer(W * 4)
    d_mel.upload(mel)
    before = _lib.kernel_launch_count()
    win.model_inputs_device(d_mel.ptr, off, frames, W, d_out.ptr, d_len.ptr, 100)
    _lib.synchronize()
    assert _lib.kernel_launch_count() - before == 1
    assert d_out.download((W, 128, 3072), np.float32).tobytes() == host_mel.tobytes()
    assert d_len.download(W, np.int32).tolist() == host_len.tolist()
    preds = K.model(host_mel, host_len)
    before = _lib.kernel_launch_count()
    host_rows, host_maps = win.stitch(preds, frames, 100, mappings=True)
    assert _lib.kernel_launch_count() - before == 1
    d_p, d_rows, d_maps = _lib.DeviceBuffer(preds.nbytes), _lib.DeviceBuffer(R * 16), _lib.DeviceBuffer(W * 16)
    d_p.upload(preds)
    before = _lib.kernel_launch_count()
    win.stitch_device(d_p.ptr, frames, d_rows.ptr, d_maps.ptr, 100)
    _lib.synchronize()
    assert _lib.kernel_launch_count() - before == 1
    assert d_rows.download((R, 4), np.float32).tobytes() == host_rows.tobytes()
    assert np.array_equal(d_maps.download((W, 4), np.int32), host_maps)
    # refusals on device buffers: nothing written
    sentinel = np.full(W * WINDOW, 7, np.float32)
    d_out.upload(sentinel)
    with pytest.raises(_lib.FluidAudioError):
        win.model_inputs_device(d_mel.ptr, off, frames, W - 1, d_out.ptr, d_len.ptr, 100)
    with pytest.raises(_lib.FluidAudioError):
        win.model_inputs_device(d_mel.ptr, off, [3001, -1, 5344, 3072, 20000], W, d_out.ptr, d_len.ptr, 100)
    _lib.synchronize()
    assert (d_out.download(W * WINDOW, np.float32) == 7).all()
    d_rows.upload(np.full(R * 4, 7, np.float32))
    with pytest.raises(_lib.FluidAudioError):
        win.stitch_device(d_p.ptr, [3001, 0, -5], d_rows.ptr, None, 100)
    _lib.synchronize()
    assert (d_rows.download(R * 4, np.float32) == 7).all()


def _segments(timeline):
    return {k: [(s.start_frame, s.end_frame, np.float32(s.activity).tobytes()) for s in sp.finalized_segments]
            for k, sp in timeline.speakers.items() if sp.finalized_segments or sp.tentative_segments}


def _oracle_segments(fin, ten):
    out = {}
    for recs in (fin, ten):
        for r in recs:
            out.setdefault(int(r["speaker"]), []).append((int(r["start_frame"]), int(r["end_frame"]),
                                                          np.float32(r["activity"]).tobytes()))
    return out


@pytest.mark.parametrize("overlap", [100, 0, 383])
def test_process_complete_batch_matches_the_oracle(overlap):
    from fluidaudio_b200.offline_sortformer import OfflineSortformerConfig
    rng = np.random.default_rng(31 + overlap)
    seconds = [0.0, 30.0, 1.0, 45.5, 0.01, 70.0] if overlap != 383 else [0.0, 30.0, 41.0]
    clips = [(rng.normal(0, 0.1, size=int(s * 16000)) * np.sin(np.arange(int(s * 16000)) / 900.0)).astype(np.float32)
             for s in seconds]
    diar = OfflineSortformerDiarizer(K.model, OfflineSortformerConfig(overlap), window_budget=3)
    got = diar.process_complete_batch(clips)
    cfg = DiarizerTimelineConfig.default(4, 0.08)
    assert cfg == diar.timeline_config
    ocfg = {k: getattr(cfg, k) for k in ("num_speakers", "frame_duration_seconds", "onset_threshold",
                                         "offset_threshold", "onset_pad_frames", "offset_pad_frames", "min_frames_on",
                                         "min_frames_off", "activity_type")}
    ocfg["max_stored_frames"] = None
    mel = AudioMelSpectrogram()
    segments = 0
    for clip, t in zip(clips, got):
        if clip.size == 0:
            assert t.speakers == {} and t.num_finalized_frames == 0 and t.state().stored.size == 0
            continue
        rows, _, nf = mel.compute_flat_transposed(clip)
        otl, fin, ten, glob = O.process_complete(rows.reshape(nf, 128), nf, overlap, K.model, ocfg)
        want = otl.state()
        st = t.state()
        assert st.finalized_frames == want.finalized_frames == glob.shape[0]
        assert st.stored.tobytes() == want.stored.tobytes() == glob.tobytes()
        assert _segments(t) == _oracle_segments(fin, ten)
        segments += len(fin) + len(ten)
    assert segments > 0
    one = diar.process_complete(clips[1])
    assert one.state().stored.tobytes() == got[1].state().stored.tobytes()


def test_process_complete_resamples_first():
    rng = np.random.default_rng(41)
    clip = rng.normal(0, 0.1, size=44100 * 12).astype(np.float32)
    diar = OfflineSortformerDiarizer(K.model)
    t = diar.process_complete(clip, source_sample_rate=44100)
    from fluidaudio_b200.audio_converter import AudioConverter
    same = diar.process_complete(AudioConverter(16000.0).resample(clip, 44100.0))
    assert t.state().stored.tobytes() == same.state().stored.tobytes() and t.num_finalized_frames > 0
