"""The prepare-stage kernels on the H100 against the oracle (``oracle/oracle_prepare.cpp``) across their configuration space:
windows, powerset decoding, the embedding plan (bit for bit on binary weights), determinism, launch counts, and the whole
chain from synthetic logits to a speaker timeline through the library's existing clustering and reconstruction calls.
"""
import itertools
import math
import threading

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.segmentation import (EmbeddingPlanConfig, OfflineEmbeddingPlanner, OfflineSegmentationProcessor,
                                          SegmentationConfig, SegmentationOutput, WeightInterpolation)

pytestmark = pytest.mark.gpu
FLT_MAX = np.finfo(np.float32).max
PLAN_FIELDS = ("chunk_index", "speaker_index", "start_frame", "end_frame", "start_time", "end_time", "mask_sum",
               "used_fallback", "reuse_of", "frame_weights", "model_weights")


@pytest.fixture(scope="module")
def P(gpu_lib):
    from oracle import oracle_prepare
    oracle_prepare.build()
    oracle_prepare.lib()
    return oracle_prepare


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def upload(a):
    buf = _lib.DeviceBuffer(max(a.nbytes, 4))
    if a.nbytes:
        buf.upload(a)
    return buf


def launches(fn):
    before = _lib.kernel_launch_count()
    out = fn()
    return _lib.kernel_launch_count() - before, out


# ---- 7. windows ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [dict(sample_rate=1000, window_duration=2.0, step_ratio=0.2),
                                 dict(sample_rate=999, window_duration=1.001, step_ratio=0.37), dict()])
def test_windows_equal_the_oracle(P, cfg):
    seg = SegmentationConfig(**cfg)
    proc = OfflineSegmentationProcessor(seg)
    _, window, step = proc.window_count(1)
    planner = OfflineEmbeddingPlanner(seg, EmbeddingPlanConfig(audio_sample_count=max(1, window - 3)))
    for total in (1, window - 1, window, window + 1, 3 * step + 7):
        audio = synth.tone_noise_audio(total, seed=total % 97)
        ref, ref_offs = P.seg_windows(audio, **{**P.SEG_DEFAULTS, **cfg})
        n, got = launches(lambda: proc.windows(audio))
        assert n == 1 and same_bits(got[0], ref) and same_bits(got[1], ref_offs)
        d_audio, d_out = upload(audio), _lib.DeviceBuffer(ref.nbytes)
        offs = proc.windows_device(d_audio, total, d_out, 0, ref.shape[0])
        assert same_bits(d_out.download(ref.shape, np.float32), ref) and same_bits(offs, ref_offs)
        if ref.shape[0] > 1:                                  # a sub-range of the windows
            part, part_offs = proc.windows(audio, 1, ref.shape[0] - 1)
            assert same_bits(part, ref[1:]) and same_bits(part_offs, ref_offs[1:])
        offsets = np.concatenate([ref_offs, [total / seg.sample_rate + 1.0, math.nan, -3.0]])
        chunks = np.arange(offsets.size + 1, dtype=np.int32)[::-1].copy()     # one chunk past the offsets: missing
        want = P.embed_windows(audio, offsets, chunks, planner.config.audio_sample_count, seg.sample_rate, seg.window_duration)
        assert same_bits(planner.fbank_windows(audio, offsets, chunks), want)
        d_rows = _lib.DeviceBuffer(want.nbytes)
        planner.fbank_windows_device(d_audio, total, offsets, chunks, chunks.size, d_rows)
        assert same_bits(d_rows.download(want.shape, np.float32), want)


# ---- 8. decode ----------------------------------------------------------------------------------------------------------
def decode_input(kind, chunks, frames, classes, rng):
    if kind == "timeline":
        x, _ = synth.segmentation_logits(2.0 * chunks, speakers=3, seed=chunks + frames, frames=frames, classes=classes)
        return np.ascontiguousarray(x[:chunks])
    x = (rng.standard_normal((chunks, frames, classes)) * 4).astype(np.float32)
    if kind == "ties":
        x = np.round(x / 4).astype(np.float32)
    elif kind == "inf":
        x[rng.random(x.shape) < 0.1] = np.inf
        x[rng.random(x.shape) < 0.2] = -np.inf
        x.reshape(-1, classes)[::5] = -np.inf
    elif kind == "nan":
        x[rng.random(x.shape) < 0.2] = np.nan
        x.reshape(-1, classes)[::7] = np.nan
        x.reshape(-1, classes)[1::7] = -FLT_MAX
    return x


def check_decode(P, x, report):
    chunks, frames, classes = x.shape
    proc = OfflineSegmentationProcessor()
    ref = P.seg_decode(x)
    n, got = launches(lambda: proc.decode(x))
    assert n == 1
    assert same_bits(got.speaker_weights, ref.speaker_weights) and same_bits(got.class_histogram, ref.class_histogram)
    # log-probabilities and the speech count: exp and log are correctly rounded on both sides (fa_float.cuh,
    # oracle_float.h), so bit for bit (NaN for NaN)
    nan = np.isnan(ref.log_probs)
    assert same_bits(np.isnan(got.log_probs), nan) and same_bits(got.log_probs[~nan], ref.log_probs[~nan])
    assert got.speech_frames == ref.speech_frames
    # the device twin leaves the same bytes on the device
    d_x, d_lp, d_w = upload(x), _lib.DeviceBuffer(x.nbytes), _lib.DeviceBuffer(ref.speaker_weights.nbytes)
    hist, speech = proc.decode_device(d_x, chunks, frames, classes, d_lp, d_w)
    assert same_bits(d_lp.download(x.shape, np.float32), got.log_probs)
    assert same_bits(d_w.download(ref.speaker_weights.shape, np.float32), got.speaker_weights)
    assert same_bits(hist, got.class_histogram) and speech == got.speech_frames
    report["frames"] += chunks * frames


def test_decode_sweep(P, capsys):
    rng = np.random.default_rng(1)
    report = dict(frames=0)
    for chunks, frames in itertools.product((1, 2, 33, 700), (1, 31, 32, 33, 589)):
        for classes in ((1, 7, 8, 11) if chunks < 700 or frames < 589 else (7,)):
            kinds = ("timeline", "random", "ties", "inf", "nan") if chunks <= 33 else ("random",)
            for kind in kinds:
                check_decode(P, decode_input(kind, chunks, frames, classes, rng), report)
    with capsys.disabled():
        print(f"\n[prepare] decode: log-probabilities and speech counts exact over {report['frames']} frames")
    without = OfflineSegmentationProcessor().decode(decode_input("random", 2, 33, 7, rng), want_log_probs=False)
    assert without.speaker_weights.shape == (2, 33, 3)


# ---- 9. plan ------------------------------------------------------------------------------------------------------------
def binary_weights(chunks, frames, speakers, rng):
    """Runs of activity per speaker with silences and overlaps; some chunks empty, some with one speaker throughout."""
    w = np.zeros((chunks, frames, speakers), np.float32)
    for c in range(chunks):
        for s in range(speakers):
            mode = rng.integers(5)
            if mode == 0:
                continue
            if mode == 1:
                w[c, :, s] = 1
                continue
            a = int(rng.integers(0, frames))
            b = int(rng.integers(a, frames + 1))
            w[c, a:b, s] = 1
            if mode == 2 and c:                              # the previous chunk's mask, slightly changed: reuse candidates
                w[c, :, s] = w[c - 1, :, s]
                w[c, int(rng.integers(frames)), s] = 1
    return w


def run_plan(seg, plan, w, offsets, fd, total):
    out = SegmentationOutput(None, w, w.shape[0], w.shape[1], w.shape[2], offsets, fd)
    return OfflineEmbeddingPlanner(seg, plan).plan(out, total)


def oracle_plan(P, seg, plan, w, offsets, fd, total):
    return P.embedding_plan(w, offsets, fd, total, dict(sample_rate=seg.sample_rate, window_duration=seg.window_duration),
                            dict(exclude_overlap=plan.exclude_overlap, min_segment_duration=plan.min_segment_duration,
                                 skip_threshold=-1.0 if plan.skip_threshold is None else plan.skip_threshold,
                                 weight_frames=plan.weight_frames, fbank_batch=plan.fbank_batch))


def assert_plans_identical(got, ref):
    assert got.count == ref.count
    for name in PLAN_FIELDS:
        assert same_bits(getattr(got, name), getattr(ref, name)), name
    assert list(got.counters.values()) == ref.counters.tolist()


def test_plan_on_binary_weights_is_bit_identical(P):
    rng = np.random.default_rng(2)
    seg = SegmentationConfig(sample_rate=1000, window_duration=10.0, step_ratio=0.2)
    seen = np.zeros(4, np.int64)
    reused = 0
    for frames, wf, speakers in itertools.product((1, 5, 589), (1, 589, 998, 1499), (1, 3, 4)):
        for exclude, thr, chunks in ((True, None, 31), (False, 0.0, 33), (True, 0.95, 70), (True, 1.0, 32)):
            w = binary_weights(chunks, frames, speakers, rng)
            offsets = np.arange(chunks - 2) * 2.0             # the last two offsets are missing
            offsets[chunks // 2] = math.nan
            offsets[3] = math.inf
            total = int(1000 * (2.0 * (chunks - 6) + 3))      # the last chunks start past the end of the audio
            fd = 0.0 if frames == 5 else 10.0 / frames
            plan = EmbeddingPlanConfig(exclude_overlap=exclude, skip_threshold=thr, weight_frames=wf,
                                       min_segment_duration=1.0 if speakers != 4 else 4.0, fbank_batch=32)
            n, got = launches(lambda: run_plan(seg, plan, w, offsets, fd, total))
            assert n == (2 if thr is None else 3)
            ref = oracle_plan(P, seg, plan, w, offsets, fd, total)
            assert_plans_identical(got, ref)
            seen += ref.counters
            reused += int((ref.reuse_of >= 0).sum())
    assert (seen > 0).all() and reused > 0, (seen, reused)


def test_plan_device_twin_and_null_outputs(P):
    rng = np.random.default_rng(3)
    seg, plan = SegmentationConfig(), EmbeddingPlanConfig(skip_threshold=0.9)
    w = binary_weights(40, 589, 3, rng)
    offsets = np.arange(40) * 2.0
    ref = oracle_plan(P, seg, plan, w, offsets, 10.0 / 589, 16000 * 90)
    cap = 40 * 3
    sizes = dict(chunk_index=4, speaker_index=4, start_frame=4, end_frame=4, start_time=8, end_time=8, mask_sum=4,
                 used_fallback=4, reuse_of=4, frame_weights=4 * 589, model_weights=4 * 589)
    d_out = {k: _lib.DeviceBuffer(cap * v) for k, v in sizes.items()}
    planner = OfflineEmbeddingPlanner(seg, plan)
    count, counters = planner.plan_device(upload(w), 40, 589, 3, offsets, 10.0 / 589, 16000 * 90, d_out)
    assert count == ref.count and list(counters.values()) == ref.counters.tolist()
    for name in PLAN_FIELDS:
        want = getattr(ref, name)
        assert same_bits(d_out[name].download(want.shape, want.dtype), want), name
    # only the weights of the embedding network and the reuse map: the masks the skip strategy compares are then the
    # library's own scratch
    few = {k: d_out[k] for k in ("model_weights", "reuse_of")}
    count2, counters2 = planner.plan_device(upload(w), 40, 589, 3, offsets, 10.0 / 589, 16000 * 90, few)
    assert (count2, counters2) == (count, counters)
    assert same_bits(few["reuse_of"].download(ref.reuse_of.shape, np.int32), ref.reuse_of)


def test_plan_on_soft_weights(P, capsys):
    """Non-binary weights: sums run in the kernel's own order, so a decision may differ from the sequential oracle where
    a sum lies within the summation bar of its threshold; every other pair decides alike, and the rows of pairs that
    chose the same mask are bit-identical."""
    rng = np.random.default_rng(4)
    seg = SegmentationConfig()
    frames, speakers, chunks, wf = 589, 3, 60, 998
    w = binary_weights(chunks, frames, speakers, rng) * rng.uniform(0.2, 1.0, (chunks, frames, speakers)).astype(np.float32)
    w[rng.random(w.shape) < 0.05] = 5e-4                      # below the activity threshold
    offsets = np.arange(chunks) * 2.0
    plan = EmbeddingPlanConfig(weight_frames=wf)
    got = run_plan(seg, plan, w, offsets, 0.0, 16000 * 200)
    ref = oracle_plan(P, seg, plan, w, offsets, 0.0, 16000 * 200)
    bar = frames * 2.0 ** -24 * frames                        # n rounding errors of at most ulp(sum) / 2, sum <= n
    min_frames = math.ceil(1.0 / (10.0 / frames))
    base, clean, energy = ref.sums[..., 0], ref.sums[..., 1], ref.sums[..., 2]
    with np.errstate(invalid="ignore"):
        near = (np.abs(base) <= bar) | (np.abs(clean - np.float32(frames) * np.float32(0.2)) <= bar) | \
            (np.abs(clean - min_frames) <= bar) | (np.abs(energy) <= bar)
    got_pairs = {(c, s): i for i, (c, s) in enumerate(zip(got.chunk_index.tolist(), got.speaker_index.tolist()))}
    ref_pairs = {(c, s): i for i, (c, s) in enumerate(zip(ref.chunk_index.tolist(), ref.speaker_index.tolist()))}
    differing = set(got_pairs) ^ set(ref_pairs)
    assert all(near[c, s] for c, s in differing), differing
    rows = 0
    for pair in set(got_pairs) & set(ref_pairs):
        i, j = got_pairs[pair], ref_pairs[pair]
        if got.used_fallback[i] != ref.used_fallback[j]:
            assert near[pair]
            continue
        assert same_bits(got.frame_weights[i], ref.frame_weights[j]) and same_bits(got.model_weights[i], ref.model_weights[j])
        assert (got.start_frame[i], got.end_frame[i], got.start_time[i], got.end_time[i]) == \
            (ref.start_frame[j], ref.end_frame[j], ref.start_time[j], ref.end_time[j])
        assert abs(float(got.mask_sum[i]) - float(ref.mask_sum[j])) <= bar
        rows += 1
    assert rows > 20
    with capsys.disabled():
        print(f"\n[prepare] soft weights: {rows} entries compared, {int(near.sum())} of {near.size} pairs within the "
              f"summation bar of a threshold, {len(differing)} decided differently")
    rows2 = rng.uniform(0, 1, (7, 589)).astype(np.float32)
    for out_len in (1, 589, 998, 300):
        assert same_bits(WeightInterpolation.resample_2d(rows2, out_len), P.weight_resample(rows2, out_len))
    assert same_bits(WeightInterpolation.zoom(rows2[0], 0.5), P.weight_resample(rows2[0], 295))


def test_plan_launch_count_does_not_depend_on_the_chunk_count():
    rng = np.random.default_rng(5)
    seg = SegmentationConfig()
    for thr, want in ((None, 2), (0.95, 3)):
        for chunks in (1, 33, 400):
            w = binary_weights(chunks, 589, 3, rng)
            n, _ = launches(lambda: run_plan(seg, EmbeddingPlanConfig(skip_threshold=thr), w, np.arange(chunks) * 2.0, 0.0,
                                             16000 * 2 * (chunks + 5)))
            assert n == want


# ---- 10. determinism ----------------------------------------------------------------------------------------------------
def test_results_are_identical_run_to_run_and_across_threads():
    """Every handle-less call leases a pooled context, so the calls of four threads interleave on contexts whose
    workspaces an earlier call of another kind has already grown: each result equals the first sequential run's."""
    from fluidaudio_b200.audio_converter import Algorithm, AudioConverter
    from fluidaudio_b200.clustering import OfflineClusterer
    from fluidaudio_b200.mel import normalize_per_feature

    rng = np.random.default_rng(6)
    logits, truth = synth.segmentation_logits(120.0, seed=8)
    chunks, frames, classes = logits.shape
    proc = OfflineSegmentationProcessor()
    planner = OfflineEmbeddingPlanner(config=EmbeddingPlanConfig(skip_threshold=0.95))
    soft = rng.uniform(0, 1, (30, 589, 3)).astype(np.float32)
    audio = synth.tone_noise_audio(16000 * 30 + 123, seed=9)
    mono = rng.uniform(-1, 1, 44100).astype(np.float32)
    planar = rng.uniform(-1, 1, (3, 48000)).astype(np.float32)
    mel = rng.standard_normal((300, 80)).astype(np.float32)
    emb, _ = synth.speaker_embeddings(200, 256, 3, seed=10)
    rho, psi = synth.synthetic_plda(emb)
    per_entry = dict(chunk_index=(np.int32, 1), speaker_index=(np.int32, 1), start_frame=(np.int32, 1),
                     end_frame=(np.int32, 1), start_time=(np.float64, 1), end_time=(np.float64, 1),
                     mask_sum=(np.float32, 1), used_fallback=(np.int32, 1), reuse_of=(np.int32, 1),
                     frame_weights=(np.float32, frames), model_weights=(np.float32, planner.config.weight_frames))

    def host_decode_and_plan():
        seg = proc.decode(logits, truth["chunk_offsets"])
        plan = planner.plan(seg, truth["total_samples"])
        soft_plan = run_plan(SegmentationConfig(), EmbeddingPlanConfig(skip_threshold=0.9), soft, np.arange(30) * 2.0, 0.0,
                             16000 * 100)
        return [seg.log_probs, seg.speaker_weights, seg.class_histogram] + \
            [getattr(p, k) for p in (plan, soft_plan) for k in PLAN_FIELDS]

    def device_decode_and_plan():
        d_lp, d_w = _lib.DeviceBuffer(logits.nbytes), _lib.DeviceBuffer(chunks * frames * 3 * 4)
        hist, speech = proc.decode_device(upload(logits), chunks, frames, classes, d_lp, d_w)
        d_out = {k: _lib.DeviceBuffer(chunks * 3 * width * np.dtype(t).itemsize) for k, (t, width) in per_entry.items()}
        count, counters = planner.plan_device(d_w, chunks, frames, 3, truth["chunk_offsets"], 10.0 / frames,
                                              truth["total_samples"], d_out)
        return [d_lp.download(logits.shape, np.float32), d_w.download((chunks, frames, 3), np.float32), hist,
                np.array([speech, count, *counters.values()])] + \
            [d_out[k].download((count, width), t) for k, (t, width) in per_entry.items()]

    steps = [
        host_decode_and_plan,
        device_decode_and_plan,
        lambda: list(proc.windows(audio)),
        lambda: [AudioConverter(algorithm=Algorithm.sinc).resample(mono, 44100)],
        lambda: [AudioConverter(algorithm=Algorithm.linear).resample_buffer(planar, 48000)],
        lambda: [normalize_per_feature(mel, 250)],
        lambda: (lambda r: [r.labels, r.initial, r.centroids])(OfflineClusterer(psi=psi).cluster(emb, rho)),
    ]

    def run(shift):   # every step, starting at step `shift`; results in step order
        order = [(k + shift) % len(steps) for k in range(len(steps))]
        out = {k: steps[k]() for k in order}
        return [a for k in range(len(steps)) for a in out[k]]

    first = run(0)
    results = [None] * 4

    def worker(i):
        _lib.set_device(0)
        results[i] = [run(i + r) for r in range(3)]

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for runs in results:
        assert runs is not None
        for again in runs:
            assert len(again) == len(first) and all(same_bits(a, b) for a, b in zip(first, again))


# ---- 11. the chain ------------------------------------------------------------------------------------------------------
def test_chain_from_logits_to_timeline_recovers_the_conversation():
    """Synthetic logits -> decode -> plan -> one embedding per entry drawn around its true speaker -> the existing
    clustering, chunk assignment and reconstruction calls: the speakers and their turn boundaries come back."""
    from fluidaudio_b200.clustering import OfflineClusterer, OfflineReconstruction, build_chunk_assignments
    speakers, duration = 3, 300.0   # a few hundred embeddings: VBx on the synthetic PLDA merges everything below that
    logits, truth = synth.segmentation_logits(duration, speakers=speakers, seed=21)
    seg = OfflineSegmentationProcessor().decode(logits, truth["chunk_offsets"])
    plan = OfflineEmbeddingPlanner().plan(seg, truth["total_samples"])
    assert plan.count > 20
    who = truth["slot_speaker"][plan.chunk_index, plan.speaker_index]
    assert (who >= 0).all()
    rng = np.random.default_rng(7)
    centres = rng.standard_normal((speakers, 256))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    emb = (centres[who] + 0.02 * rng.standard_normal((plan.count, 256))).astype(np.float32)
    rho, psi = synth.synthetic_plda(emb)
    prepared = plan.to_prepared(emb, rho)
    assert prepared.embedding_count == plan.count and prepared.segmentation_chunk_count == seg.num_chunks
    res = OfflineClusterer(psi=psi).cluster(emb, rho, chunk_indices=plan.chunk_index)
    labels = res.labels
    k = int(labels.max()) + 1
    assert k == speakers
    mapping = {}
    for lab, true in zip(labels.tolist(), who.tolist()):    # every cluster is one true speaker
        assert mapping.setdefault(lab, true) == true
    assert len(set(mapping.values())) == speakers
    hard = build_chunk_assignments(plan.chunk_index, plan.speaker_index, labels, seg.num_chunks, seg.num_speakers, k)
    segments = OfflineReconstruction(seg.frame_duration, min_segment_duration=0.0).build_segments(
        seg.speaker_weights, hard, k, seg.chunk_offsets)
    assert segments
    # outside overlaps (and away from them by a frame), the reconstructed speaker at a turn's midpoint is the turn's
    # speaker, and each turn boundary that borders silence is met within one frame by a segment of that speaker
    fd = seg.frame_duration
    turns = truth["turns"]

    def speakers_at(t):
        return {mapping[s.cluster] for s in segments if s.start_time_seconds <= t < s.end_time_seconds}

    def truly_at(t):
        return {int(w) for w, a, b in turns if a <= t < b}

    checked = 0
    for w_, a, b in turns:
        mid = 0.5 * (a + b)
        if truly_at(mid) == {int(w_)} and b - a > 1.5:
            assert int(w_) in speakers_at(mid), (w_, a, b)
            checked += 1
        for edge, inside in ((a, a + 3 * fd), (b, b - 3 * fd)):
            alone = truly_at(edge - 3 * fd) | truly_at(edge + 3 * fd) == {int(w_)}
            if alone and b - a > 1.5 and 3 * fd < edge < duration - 3 * fd:
                near = [s for s in segments if mapping[s.cluster] == int(w_) and
                        min(abs(s.start_time_seconds - edge), abs(s.end_time_seconds - edge)) <= 1.5 * fd]
                assert near, (w_, a, b, edge)
                checked += 1
    assert checked > 10
