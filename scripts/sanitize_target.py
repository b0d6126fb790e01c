"""Small end-to-end pass over every kernel for compute-sanitizer (memcheck / racecheck / synccheck)."""
import sys
import numpy as np
sys.path.insert(0, ".")
from fluidaudio_b200 import synth, clustering as cl
import os
from fluidaudio_b200.mel import (AudioMelSpectrogram, LSEENDMelFrontend, UnifiedMelExtractor, PaddingMode, Precision,
                                 normalize_per_feature)
from fluidaudio_b200.audio_converter import AudioConverter

a = synth.tone_noise_audio(16000 * 3 + 77)
for nm in (80, 128):
    m = AudioMelSpectrogram(n_mels=nm)
    m.compute_flat_transposed(a)
    m.compute_flat(a[:20001])
    m.compute_flat_transposed(a[:9000], padding_mode=PaddingMode.pre_padded)
    m.compute(a[:4000])
# round 2: float32-pair transform, any-nFFT kernel, converter stage (sinc / linear / mixdown), fused PCM -> mel
m = AudioMelSpectrogram(n_mels=80, precision=Precision.f32)
m.compute_flat_transposed(a)
m.compute_flat(a[:20001])
m.compute_flat_transposed(a[:161])
for kw in (dict(n_fft=256, win_length=200, hop_length=80, n_mels=23), dict(n_fft=1024, win_length=800, hop_length=321, n_mels=64)):
    g = AudioMelSpectrogram(**kw)
    g.compute_flat_transposed(a[:30000])
    g.compute_flat(a[:5000])
conv = AudioConverter()
t = np.arange(48000) / 48000.0
st = np.stack([np.sin(2 * np.pi * 440 * t), np.sin(2 * np.pi * 550 * t)]).astype(np.float32)
conv.resample(st[0], 48000)
conv.resample(st[0][:22050], 22050)
conv.resample_buffer(np.round(st * 32767).astype(np.int16), 44100)
conv.resample_buffer(np.stack([st[0], st[1], st[0], st[1]])[:, :8000], 8000)
conv.resample_buffer(st[:, :16000], 16000)
# sinc: 32-bit phases on the interpolated path, 64-bit phases (44100.001 Hz), the largest accepted ratio (opt-in shared
# memory), an odd H (padded rows) with a non-finite sample
conv.resample(st[0][:16001], 16001)
conv.resample(st[0][:44100], 44100.001)
conv.resample(np.tile(st[0], 4)[:16000 * 168 // 4], 16000 * 168)
nan_in = st[0][:8820].copy()
nan_in[4000] = np.nan
conv.resample(nan_in, 44100)
m.compute_from_pcm(np.ascontiguousarray(np.round(st.T * 32767).astype(np.int16)), 48000, interleaved=True)
m.compute_from_pcm(np.round(st[0] * 32767).astype(np.int16)[:16000], 16000)
UnifiedMelExtractor(24000).features(np.concatenate([a[:20000], np.zeros(4000, np.float32)]), 20000)
LSEENDMelFrontend().process(a[:16000])
# adapters: a partial last 128-bin CTA and a partial last 32-frame tile with one valid frame, LS-EEND on the 8 kHz model's
# configuration (nFFT 256, the any-nFFT kernel), the standalone normalisation across two CTAs
UnifiedMelExtractor(50 * 160 + 37, n_mels=257).features(a[:50 * 160 + 37], 160)
LSEENDMelFrontend(n_fft=256, hop_length=80, win_length=200, sample_rate=8000).process(a[:8000])
normalize_per_feature(np.random.default_rng(0).normal(size=(45, 129)).astype(np.float32), 40)
for n in (2, 3, 50, 400):
    emb, _ = synth.speaker_embeddings(n, 256, 4, seed=n)
    rho, psi = synth.synthetic_plda(emb)
    chunk = (np.arange(n) // 2).astype(np.int32)
    cl.OfflineClusterer(psi=psi).cluster(emb, rho)
    cl.OfflineClusterer(psi=psi).cluster(emb, rho, chunk_indices=chunk)
    if n >= 50:
        cl.OfflineClusterer(cl.OfflineDiarizerConfig().with_speakers(exactly=6), psi=psi).cluster(emb, rho)
# hundreds of speakers: E-step reads alpha through L2; batch entry point: several sets side by side
rng = np.random.default_rng(0)
emb, _ = synth.speaker_embeddings(320, 256, 4, seed=5)
rho, psi = synth.synthetic_plda(emb)
init = np.concatenate([np.arange(260), rng.integers(0, 260, 60)]).astype(np.int32)
vbx = cl.VBxClustering(psi=psi).refine(rho, init)
# the standalone clustering entry points, each on its own scratch arena: normalisation, AHC, K-Means (identity and
# n_init runs), centroids on both sides of the fused-path limit (64 speakers), assignment with and without scores
x = emb.astype(np.float64)
cl.l2_normalize_rows(x)
cl.AHCClustering().cluster(x[:120], 0.6)
cl.KMeansClustering.cluster_with_centroids_n_init(x, 6, max_iterations=20, n_init=3)
cl.KMeansClustering.cluster_with_centroids_n_init(x[:5], 6)
cents = cl.compute_centroids(x, vbx)
small = cl.VBxClustering(psi=psi).refine(rho, init % 8)
cl.compute_centroids(x, small)
cl.assign_embeddings(x, cents)
cl.assign_embeddings(x, cents[:7], want_scores=True)
emb, _ = synth.speaker_embeddings(900, 256, 4, seed=6)
rho, psi = synth.synthetic_plda(emb)
cl.OfflineClusterer(psi=psi).cluster_batch(emb, rho, np.array([0, 300, 600, 900], np.int64))
m = AudioMelSpectrogram(n_mels=80)
m.compute_batch([a[:30000], a[:1000], a[:48077]])
# the float32 filter of the AHC nearest-neighbour pass is on from N = 2048 (FA_AHC_FILTER_MIN_N lowers it for this run)
emb, _ = synth.speaker_embeddings(700, 64, 3, seed=8)
cl.centroid_linkage(emb.astype(np.float64))
# merge kernel placements (ahc_placement.h): master heap + nn in shared memory (level 2), and node vectors streamed in two
# rounds per scan thread with the heap alone in shared memory (level 1; two rounds on 131 worker CTAs)
cl.centroid_linkage(rng.standard_normal((12000, 4)))
cl.centroid_linkage(rng.standard_normal((16769, 4)))
# pipeline branches: a non-finite rho row (every E-step row falls back to uniform gamma), AHC refusing D = 7 197
# (identity labels, one speaker per row), and a batch with empty sets at the start, the middle and the end
emb, _ = synth.speaker_embeddings(300, 256, 4, seed=10)
rho, psi = synth.synthetic_plda(emb)
rho[5, 3] = np.nan
cl.OfflineClusterer(psi=psi).cluster(emb, rho, chunk_indices=(np.arange(300) // 2).astype(np.int32))
wide, _ = synth.speaker_embeddings(40, 7197, 3, seed=11)
cl.OfflineClusterer().cluster(wide, rng.standard_normal((40, 16)))
emb, _ = synth.speaker_embeddings(900, 256, 4, seed=12)
rho, psi = synth.synthetic_plda(emb)
cl.OfflineClusterer(psi=psi).cluster_batch(emb, rho, np.array([0, 0, 300, 300, 600, 900, 900], np.int64))
# torch-style frontends: the any-nFFT kernel's reflect / magnitude / affine variants on clips shorter than the pad, the
# Cohere table on mel512_kernel with its CMVN epilogue (padOrTruncate both ways), and a general spectrum power
from fluidaudio_b200.mel import CohereMelSpectrogram, LuxTtsMelExtractor, StyleTTS2MelExtractor
b = synth.tone_noise_audio(24000 * 2 + 5)
sty, lux = StyleTTS2MelExtractor(), LuxTtsMelExtractor()
for n in (0, 1, 700, 24000 * 2 + 5):
    sty.compute(b[:n])
    lux.extract(b[:n])
coh = CohereMelSpectrogram()
coh.features(a[:16000 * 3], 100)
coh.features(a[:1000], 3500)
coh.compute(a[:1])
CohereMelSpectrogram(CohereMelSpectrogram.Config(mag_power=1.5)).compute(a[:5000])
sty.mel.compute_batch([b[:3], b[:30000]])
# host-buffer staging: the prepare stage, live mel streams, Sortformer sessions and timelines, host and device variants
# alternating on seeded inputs (outputs of the embedding plan partly null, with and without the skip strategy)
import ctypes as C
from fluidaudio_b200 import _lib
from fluidaudio_b200.diarizer_timeline import SEGMENT, DiarizerTimelineConfig, DiarizerTimelines
from fluidaudio_b200.mel import MelStreams
from fluidaudio_b200.segmentation import (EmbeddingPlanConfig, OfflineEmbeddingPlanner, OfflineSegmentationProcessor,
                                          WeightInterpolation)
from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams


keep = []   # device buffers live until the end: the device variants return with their work queued


def dev(x=None, nbytes=0):
    d = _lib.DeviceBuffer(nbytes if x is None else x.nbytes)
    if x is not None:
        d.upload(x)
    keep.append(d)
    return d


rng = np.random.default_rng(21)
speech = (rng.standard_normal(16000 * 25 + 311) * 0.1).astype(np.float32)
segp, planner = OfflineSegmentationProcessor(), OfflineEmbeddingPlanner()
_, offs = segp.windows(speech, 1, 3)
segp.windows_device(dev(speech), speech.size, _lib.DeviceBuffer(3 * 160000 * 4), 1, 3)
planner.fbank_windows(speech, offs)
planner.fbank_windows_device(dev(speech), speech.size, offs, np.array([2, 0], np.int32), 2,
                             _lib.DeviceBuffer(2 * 160000 * 4))
logits, truth = synth.segmentation_logits(30.0, seed=4)
seg = segp.decode(logits, truth["chunk_offsets"])
segp.decode(logits, truth["chunk_offsets"], want_log_probs=False)
c, f, k = logits.shape
d_logits, d_w = dev(logits), _lib.DeviceBuffer(c * f * 3 * 4)
segp.decode_device(d_logits, c, f, k, _lib.DeviceBuffer(logits.nbytes), d_w)
segp.decode_device(d_logits, c, f, k, None, d_w)
planner.plan(seg, truth["total_samples"])
for skip in (None, 0.9):
    cfg = EmbeddingPlanConfig(skip_threshold=skip)
    pairs, wf = c * 3, cfg.weight_frames
    d_out = {"chunk_index": _lib.DeviceBuffer(pairs * 4), "start_time": _lib.DeviceBuffer(pairs * 8),
             "reuse_of": _lib.DeviceBuffer(pairs * 4), "model_weights": _lib.DeviceBuffer(pairs * wf * 4)}
    OfflineEmbeddingPlanner(config=cfg).plan_device(dev(seg.speaker_weights), c, f, 3, seg.chunk_offsets,
                                                    seg.frame_duration, truth["total_samples"], d_out)
    ci, st, ro, mw = np.zeros(pairs, np.int32), np.zeros(pairs), np.zeros(pairs, np.int32), np.zeros((pairs, wf), np.float32)
    n, counters = C.c_int32(), np.zeros(4, np.int64)
    _lib.check(_lib.load().fa_embedding_plan(
        _lib.ptr(seg.speaker_weights), c, f, 3, _lib.ptr(seg.chunk_offsets), c, float(seg.frame_duration),
        int(truth["total_samples"]), C.byref(segp.config._c()), C.byref(cfg._c()), _lib.ptr(ci), None, None, None,
        _lib.ptr(st), None, None, None, _lib.ptr(ro), None, _lib.ptr(mw), C.byref(n), counters.ctypes.data),
        "fa_embedding_plan")
WeightInterpolation.resample_2d(rng.random((5, 589), np.float32), 293)
mel = AudioMelSpectrogram(n_mels=80)
ms = MelStreams(mel)
s1, s2 = ms.open(), ms.open()
for i, n in enumerate((700, 2500, 0, 4001)):
    if i % 2 == 0:
        ms.push({s1: speech[i * 5000:i * 5000 + n], s2: speech[:n + 160]})
    else:
        offsets = np.array([0, n, 2 * n + 160], np.int64)
        rows = ms.pending_frames(s1, n) + ms.pending_frames(s2, n + 160)
        ms.push_device([s1, s2], dev(np.concatenate([speech[:n], speech[:n + 160]])), offsets,
                       dev(nbytes=max(rows, 1) * 80 * 4))
ms.push({s1: speech[:333]}, finish=[s1, s2])
sf = SortformerStreams(SortformerConfig.preset("default"))
ids = [sf.open() for _ in range(3)]
conf_d, tent_d = _lib.DeviceBuffer(3 * 6 * 4 * 4), _lib.DeviceBuffer(16)
sc_d, ff_d = _lib.DeviceBuffer(3 * 188 * 512 * 4), _lib.DeviceBuffer(3 * 40 * 512 * 4)
for step in range(45):   # past the speaker cache's first compression
    e = (rng.standard_normal((3, 6, 512)) * 0.5).astype(np.float32)
    p = rng.random((3, 240, 4), np.float32)
    if step % 2 == 0:
        sf.update(ids, e, p, left_context=0, right_context=0)
        sf.model_inputs(ids[:2])
    else:
        sf.update_device(ids, dev(e), 6, dev(p), 240, conf_d, tent_d, left_context=0, right_context=0)
        sf.model_inputs_device(ids[1:], sc_d, ff_d)
_lib.synchronize()
tl = DiarizerTimelines(DiarizerTimelineConfig.sortformer_default(), max_tentative_rows=64)
tids = [tl.open_session() for _ in range(2)]
for step in range(4):
    fin = [rng.random((r, 4), np.float32) for r in (40, 17)]
    ten = [rng.random((r, 4), np.float32) for r in (8, 0)]
    if step % 2 == 0:
        tl.push(tids, fin, ten)
    else:
        fr, tr = [40, 17], [8, 0]
        bf, bt = tl.segment_bound(fr, tr)
        tl.push_device(tids, dev(np.concatenate(fin)), fr, dev(np.concatenate(ten)), tr,
                       dev(nbytes=max(bf, 1) * SEGMENT.itemsize), dev(nbytes=max(bt, 1) * SEGMENT.itemsize), dev(nbytes=16),
                       dev(nbytes=16))
tl.finalize(tids)
tl.reset(tids[:1])
tl.push(tids, [rng.random((9, 4), np.float32)] * 2)
# CTC decoding: greedy over three clips, beam search with a small bigram LM (the radix select, the parent fold-in, the
# trie conses, the LM walk), beam_width 0 and the NaN refusal
from fluidaudio_b200 import ctc_decoding as CD
crng = np.random.default_rng(21)
cvoc = {v: ("\u2581" if v % 3 == 0 else "") + "ab"[v % 2] + "cd"[(v // 2) % 2] for v in range(16)}
cclips = [np.round(crng.normal(0, 1, size=(T, 17)) * 2).astype(np.float32) / 2 - 3 for T in (30, 0, 11)]
CD.greedy_ids(cclips, 17, 16)
carpa = CD.ARPALanguageModel()
carpa.unigrams = {w: CD.ARPALanguageModel.Entry(np.float32(-1.5), np.float32(-0.3)) for w in ("ac", "bd", "acbd")}
carpa.bigrams = {"ac": {"bd": CD.ARPALanguageModel.Entry(np.float32(-0.2), np.float32(0.0))}}
cdec = CD.CtcDecoder(cvoc, 17, 16)
cdec.beam_search(cclips, carpa, 8, 0.3, 0.1, 5)
cdec.beam_search(cclips, None, 0, 0.3, 0.0, 5)
cbad = [cclips[0].copy()]
cbad[0][3, 2] = np.nan
try:
    cdec.beam_search(cbad, carpa, 8, 0.3, 0.1, 5)
except _lib.FluidAudioError:
    pass
cdec.close()
# VAD: Silero sessions with chunks of 0, 1, 63, 64, 4096 and 5000 samples (host and device), a refused advance,
# segmentation of clips with split corners, and the FSMN decision
from fluidaudio_b200 import vad as VD
vrng = np.random.default_rng(22)
vst = VD.SileroVadStreams()
vids = [vst.open() for _ in range(6)]
for _ in range(3):
    vin, vh, vc = vst.model_inputs(vids, [vrng.normal(size=n).astype(np.float32) for n in (0, 1, 63, 64, 4096, 5000)])
    vst.advance(vids, vrng.uniform(size=6).astype(np.float32), vh + 1, vc - 1,
                seg=VD.VadSegmentationConfig(min_silence_duration=0.0))
try:
    vst.advance(vids[:1], [0.5], vh[:1], vc[:1])
except _lib.FluidAudioError:
    pass
vaud = _lib.DeviceBuffer(4096 * 4)
vbuf = [_lib.DeviceBuffer(n) for n in (4160 * 4, 128 * 4, 128 * 4)]
vst.model_inputs_device(vids[:1], vaud, np.array([0, 4096], np.int64), *vbuf)
vst.state(vids[0])
vst.close_handle()
vprobs = [np.repeat(vrng.choice(np.array([0.1, 0.5, 0.9], np.float32), size=n), 4)[:4 * n] for n in (0, 5, 300)]
VD.segment_sample_ranges(vprobs, [0, 20000, 300 * 4096], seg=VD.VadSegmentationConfig(max_speech_duration=2.0))
VD.fsmn_vad_decide([np.repeat(vrng.choice(np.array([0.05, 0.9], np.float32), size=50), 90) for _ in range(3)])
# online diarization: model inputs (chunks of 0 to 200 000 samples, enrollment), two sessions over four chunks with
# databases grown past a reallocation, the database operations, queries, a refused advance and the device variants
from fluidaudio_b200 import online_diarizer as ODZ
orng = np.random.default_rng(23)
ODZ.chunk_inputs([orng.normal(size=n).astype(np.float32) for n in (0, 1, 80000, 200000)])
ODZ.enrollment_inputs([orng.normal(size=n).astype(np.float32) for n in (0, 100, 170000)], 589)
odb = ODZ.SpeakerDatabases(589, ODZ.DiarizerConfig(min_speech_duration=0.1))
oids = [odb.open() for _ in range(2)]
odb.initialize_known_speakers(oids[0], [ODZ.Speaker(str(k), orng.normal(size=256).astype(np.float32), 1.0, 1,
                                                    orng.normal(size=(3, 256)).astype(np.float32)) for k in range(6)])
for t in range(4):
    olg = np.repeat(np.eye(7, dtype=np.float32)[orng.integers(0, 7, size=(2, 31))], 19, axis=1)[:, :589] * 4
    odb.embedding_inputs(oids, olg)
    odb.advance(oids, orng.normal(size=(2, 3, 256)).astype(np.float32), [10.0 * t] * 2)
odb.upsert_speaker(oids[1], ODZ.Speaker("alice", orng.normal(size=256).astype(np.float32), 2.0))
odb.merge_speaker(oids[0], "1", "2")
odb.set_permanent(oids[0], "3")
odb.remove_speaker(oids[0], "4")
odb.find_mergeable_pairs(oids[0], 2.0)
odb.find_matching_speakers(oids[1], orng.normal(size=256).astype(np.float32), 2.0)
try:
    odb.advance(oids, np.zeros((2, 3, 256), np.float32), [0.0, 0.0])
except _lib.FluidAudioError:
    pass
odb.reset(oids[0], True)
odb.speakers(oids[0])
odb.close_handle()
# LuxTTS: begin with boosted and unboosted prompts (one capped) and a refused call, a text condition at row stride 112,
# four interleaved steps, the vocoder input at both buckets and finish with its capacity refusal
from fluidaudio_b200 import luxtts as LX
lrng = np.random.default_rng(24)
lreq = LX.LuxTtsRequests()
lprompts = [(lrng.normal(size=n) * s).astype(np.float32) for n, s in ((30000, 0.02), (130000, 0.3), (5000, 0.2))]
lids, lplans, _, _ = lreq.begin(lprompts, [40, 60, 10], [50, 120, 30], [1.0, 1.0, 1.0], [0, 1, 2])
try:
    lreq.begin([lprompts[0], np.zeros(3000, np.float32)], [5, 5], [5, 5], [1.0, 1.0], [3, 4])
except LX.LuxTtsError:
    pass
lreq.text_condition(lids, lrng.normal(size=(3, 256, 112)).astype(np.float32))
for k in range(4):
    lsel = lids if k % 2 == 0 else lids[::-1]
    lreq.model_inputs(lsel)
    lreq.advance(lsel, lrng.normal(size=(3, 1024, 100)).astype(np.float32))
for lb in (282, 555):
    lsel = np.array([r for r, p in zip(lids, lplans) if p.bucket == lb], np.int32)
    if lsel.size:
        lreq.vocoder_input(lsel, lb)
        lreq.finish(lsel, lrng.normal(size=(lsel.size, (lb - 1) * 512)).astype(np.float32))
lreq.close_handle()
# StyleTTS2 glue: sampler inputs for two buckets and a refusal, the blend, align at odd widths and its too-small and
# NaN refusals
from fluidaudio_b200 import styletts2 as ST
srng = np.random.default_rng(25)
sglue = ST.StyleTTS2Glue()
sglue.sampler_inputs([srng.integers(0, 178, size=k) for k in (3, 57)], [0, 1], 57)
sglue.sampler_inputs([srng.integers(0, 178, size=k) for k in (65, 128)], [2, 3], 128)
try:
    sglue.sampler_inputs([np.zeros(3, np.int32), np.zeros(64, np.int32)], [0, 0], 57)
except _lib.FluidAudioError:
    pass
sglue.blend_style(srng.normal(size=(3, 256)), srng.normal(size=(3, 256)), [0.3, 1.0, 0.0], [0.7, 0.0, 1.0])
scounts = (1, 40, 256)
slog = [srng.normal(size=(k, 4)).astype(np.float32) * 3 for k in scounts]
sd = [srng.normal(size=(k, 33)).astype(np.float32) for k in scounts]
st_en = [srng.normal(size=(3, k)).astype(np.float32) for k in scounts]
sglue.align(slog, sd, st_en)
try:
    sglue.align(slog, sd, st_en, frame_stride=2)
except _lib.FluidAudioError:
    pass
slog[1][5, 2] = np.nan
try:
    sglue.align(slog, sd, st_en, frame_stride=2000)
except ST.StyleTTS2Error:
    pass
# offline Sortformer windows: model inputs and the stitch at three overlaps, an empty file and a refusal
from fluidaudio_b200 import offline_sortformer as OSF
orng = np.random.default_rng(26)
owin = OSF.OfflineSortformerWindows()
for oov in (0, 100, 383):
    oframes = [1, 3072, 0, 5344]
    omel = orng.normal(size=sum(oframes) * 128).astype(np.float32)
    ooff = np.concatenate([[0], np.cumsum(oframes)])[:-1] * 128
    oin, olen = owin.model_inputs(omel, ooff, oframes, oov)
    owin.stitch(orng.random((olen.size, 384, 4), np.float32), oframes, oov, mappings=True)
try:
    owin.stitch(np.zeros(384 * 4, np.float32), [3, -1], 100)
except _lib.FluidAudioError:
    pass
_lib.synchronize()
print("sanitize target done")
