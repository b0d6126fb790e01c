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
print("sanitize target done")
