"""``fa_kernel_launch_count``: every launch is counted where it is issued, and the count of each entry point follows
from its code.

The CPU test checks that every kernel launch under ``fluidaudio_b200/csrc/`` goes through the counting helpers of
``fa_common.cuh`` (``fa::launch`` / ``fa::launch_cooperative``), so a new kernel cannot be left out of the count.  The
GPU tests restate, per entry point, which kernels its host code launches for small seeded inputs and compare that with
the counter's delta (the VBx formula follows ``tests/test_gpu_cluster_sweep.py``).
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from csrc_sources import path, sources  # noqa: E402


def _code(path):
    """source text without comments"""
    with open(path, encoding="utf-8") as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return re.sub(r"//[^\n]*", " ", text)


def test_every_launch_goes_through_the_counting_helpers():
    offenders = []
    for name in sources():
        if name == "fa_common.cuh":
            continue
        code = _code(path(name))
        for token in ("<<<", "cudaLaunchCooperativeKernel", "cudaLaunchKernel"):
            if token in code:
                offenders.append(f"{name}: {token}")
    assert not offenders, f"launches outside fa::launch / fa::launch_cooperative: {offenders}"


# ---- GPU: launch-count deltas of each entry point ------------------------------------------------------------------
FILTER_MIN_N = int(os.environ.get("FA_AHC_FILTER_MIN_N", "2048"))   # ahc_kernels.cu hooks(): the float32 filter
K_ETHREADS, K_FUSED_MAX_S, SMEM = 128, 64, 200 * 1024                  # vbx_kernels.cu
MEL_UNITS, MEL_MIN_UNIT, TILE_FRAMES = 24, 4096, 16                    # mel_plan.h pipeline_chunks, compute_host


def _delta(fn):
    from fluidaudio_b200 import _lib
    before = _lib.kernel_launch_count()
    out = fn()
    return _lib.kernel_launch_count() - before, out


def mel_units(T, max_units=MEL_UNITS, min_unit=MEL_MIN_UNIT):
    """MelPlan::compute_host's unit count (unit_bounds): one mel launch per unit"""
    K = max(1, min(max_units, T // max(1, min_unit)))

    def weight(c, k):
        if k < 6:
            return 4
        e = min(c, k - 1 - c)
        return 1 if e == 0 else (2 if e == 1 else 4)

    while K > 1 and T * weight(0, K) // sum(weight(c, K) for c in range(K)) < min_unit:
        K -= 1
    total = sum(weight(c, K) for c in range(K))
    b, acc = [0], 0
    for c in range(K - 1):
        acc += weight(c, K)
        e = min(T, -(-int(T * acc / total) // TILE_FRAMES) * TILE_FRAMES)
        if b[-1] < e < T:
            b.append(e)
    return len(b)


def vbx_launches(S, D, max_it):
    fused = S <= K_FUSED_MAX_S and 8 * (S * D + 2 * S + K_ETHREADS * S + K_ETHREADS) <= SMEM
    if fused:
        return 3 if max_it == 0 else 2 * max_it + 4   # init, partials0, (update2, estep2) x max_it, closing update2, hard
    return 4 * max_it + 2                             # init, (accumulate, update, estep, finish) x max_it, hard


def ahc_launches(N):
    """linkage_device: stage, the initial nearest-neighbour pass (exact: 2; float32 filter: 6), merge"""
    return 1 + (6 if 0 < FILTER_MIN_N <= N else 2) + 1


def centroid_launches(S):
    return 3 if S <= K_FUSED_MAX_S else 2


def kmeans_launches(N, k, max_it, n_init):
    """cluster_ninit_device with max_it <= 8 (one polling batch per run)"""
    if N <= k:
        return 1
    runs = n_init if n_init > 1 else 1
    return 2 + runs * (1 + 3 * max_it + 2)


@pytest.fixture
def mel(gpu_lib):
    from fluidaudio_b200.mel import AudioMelSpectrogram
    m = AudioMelSpectrogram(n_mels=80)
    yield m
    m.close()


@pytest.mark.gpu
def test_resample(gpu_lib):
    from fluidaudio_b200 import _lib
    x = np.sin(np.arange(2 * 4410) * 0.05).astype(np.float32)
    for in_rate, channels, algorithm in ((16000.0, 2, 0), (44100.0, 1, 2), (44100.0, 1, 1)):   # mixdown, linear, sinc
        fmt = _lib.AudioFormat(in_rate, 16000.0, channels, 0, 0, algorithm)
        frames = x.size // channels
        n = int(gpu_lib.fa_resample_output_count(C.byref(fmt), frames))
        out, cnt = np.zeros(n, np.float32), C.c_int64()
        d, _ = _delta(lambda: _lib.check(gpu_lib.fa_audio_resample(x.ctypes.data, frames, C.byref(fmt), out.ctypes.data,
                                                                    n, C.byref(cnt)), "fa_audio_resample"))
        assert d == 1, (in_rate, channels, algorithm, d)


@pytest.mark.gpu
def test_mel_host_buffer(mel):
    from fluidaudio_b200 import synth
    a = synth.tone_noise_audio(16000 * 180 + 77)
    for n in (16000, a.size):
        T = mel.frame_count(n)
        d, _ = _delta(lambda: mel.compute_flat_transposed(a[:n]))
        assert d == mel_units(T), (n, T, d)
    assert mel_units(mel.frame_count(a.size)) > 1
    pcm = np.round(a[:16000] * 32767).astype(np.int16)
    d, _ = _delta(lambda: mel.compute_from_pcm(pcm, 16000))          # one unit: conversion + mel
    assert d == 2
    d, _ = _delta(lambda: mel.compute_from_pcm(a[:48000], 48000))    # one unit: sinc + mel
    assert d == 2


@pytest.mark.gpu
def test_mel_device_and_batch(mel):
    from fluidaudio_b200 import _lib, synth
    a = synth.tone_noise_audio(48077)
    d_a, d_o = _lib.DeviceBuffer(4 * a.size), _lib.DeviceBuffer(4 * 80 * 400)
    d_a.upload(a)
    d, _ = _delta(lambda: (mel.compute_device(d_a, 20000, d_o), _lib.synchronize()))
    assert d == 1
    clips = [a[:30000], a[:0], a[:1000], a[:48077]]                   # the empty clip's group launches nothing
    d, _ = _delta(lambda: mel.compute_batch(clips))
    assert d == 3
    offsets = np.array([0, 9000, 9000, 20000, 30001], np.int64)
    out_offsets = np.zeros(offsets.size, np.int64)
    for i in range(offsets.size - 1):
        out_offsets[i + 1] = out_offsets[i] + max(1, mel.frame_count(int(offsets[i + 1] - offsets[i]))) * 80
    d_o2 = _lib.DeviceBuffer(4 * int(out_offsets[-1]))
    d, _ = _delta(lambda: (mel.compute_batch_device(d_a, offsets, d_o2, out_offsets), _lib.synchronize()))
    assert d == 1
    for b in (d_a, d_o, d_o2):
        b.free()


@pytest.mark.gpu
def test_mel_adapters(gpu_lib):
    from fluidaudio_b200 import synth
    from fluidaudio_b200.mel import LSEENDMelFrontend, UnifiedMelExtractor, normalize_per_feature
    a = synth.tone_noise_audio(24000)
    u = UnifiedMelExtractor(24000)
    assert _delta(lambda: u.features(a, 20000))[0] == 2              # mel + normalisation epilogue
    assert _delta(lambda: u.features(a, 0))[0] == 1                  # no valid frame: mel only
    assert _delta(lambda: LSEENDMelFrontend().process(a[:16000]))[0] == 2
    x = np.random.default_rng(0).normal(size=(50, 80)).astype(np.float32)
    assert _delta(lambda: normalize_per_feature(x, 30))[0] == 1
    assert _delta(lambda: normalize_per_feature(x, 0))[0] == 0


def _norm_rows(gpu_lib, x):
    from fluidaudio_b200 import _lib
    out = np.zeros_like(x)
    _lib.check(gpu_lib.fa_l2_normalize_rows(x.ctypes.data, x.shape[0], x.shape[1], out.ctypes.data), "normalize")
    return out


def _ahc(gpu_lib, x, threshold=0.6):
    from fluidaudio_b200 import _lib
    labels = np.zeros(x.shape[0], np.int32)
    _lib.check(gpu_lib.fa_ahc_cluster(x.ctypes.data, x.shape[0], x.shape[1], threshold, labels.ctypes.data), "ahc")
    return labels


@pytest.mark.gpu
def test_normalize_and_ahc(gpu_lib):
    rng = np.random.default_rng(1)
    x = rng.normal(size=(300, 32))
    assert _delta(lambda: _norm_rows(gpu_lib, x))[0] == 1
    for n in (300, max(FILTER_MIN_N, 2) + 52):
        x = rng.normal(size=(n, 32))
        d, _ = _delta(lambda: _ahc(gpu_lib, x))
        assert d == 1 + ahc_launches(n), (n, d)


def _kmeans(gpu_lib, x, k, max_it, n_init, seed=0):
    from fluidaudio_b200 import _lib
    N, D = x.shape
    labels, cent = np.zeros(N, np.int32), np.zeros((k, D))
    rows, best = C.c_int32(), C.c_int32()
    _lib.check(gpu_lib.fa_kmeans_cluster(x.ctypes.data, N, D, k, max_it, n_init, seed, labels.ctypes.data,
                                         cent.ctypes.data, k, C.byref(rows), C.byref(best)), "fa_kmeans_cluster")
    return labels


@pytest.mark.gpu
def test_kmeans(gpu_lib):
    x = np.random.default_rng(2).normal(size=(200, 16))
    for max_it in (1, 8):
        for n_init in (1, 4):
            d, _ = _delta(lambda: _kmeans(gpu_lib, x, 5, max_it, n_init))
            assert d == kmeans_launches(200, 5, max_it, n_init), (max_it, n_init, d)
    assert _delta(lambda: _kmeans(gpu_lib, x[:4], 5, 8, 4))[0] == kmeans_launches(4, 5, 8, 4)


@pytest.mark.gpu
def test_centroids_and_assignment(gpu_lib):
    from fluidaudio_b200 import _lib
    rng = np.random.default_rng(3)
    T, dim = 300, 32
    emb = rng.normal(size=(T, dim))
    for S in (8, K_FUSED_MAX_S + 6):
        gamma = rng.random((T, S)) + 0.01
        gamma /= gamma.sum(1, keepdims=True)
        pi = gamma.sum(0) / T
        cent, K = np.zeros((S, dim)), C.c_int32()
        d, _ = _delta(lambda: _lib.check(gpu_lib.fa_compute_centroids(emb.ctypes.data, T, dim, gamma.ctypes.data,
                                                                       pi.ctypes.data, S, cent.ctypes.data, C.byref(K)),
                                         "fa_compute_centroids"))
        assert d == centroid_launches(S), (S, d)
    cent = rng.normal(size=(6, dim))
    labels, scores = np.zeros(T, np.int32), np.zeros((T, 6))
    d, _ = _delta(lambda: _lib.check(gpu_lib.fa_assign_embeddings(emb.ctypes.data, T, dim, cent.ctypes.data, 6,
                                                                   labels.ctypes.data, scores.ctypes.data), "assign"))
    assert d == 2   # centroid normalisation + assignment


def _cluster(gpu_lib, emb, rho, psi, cfg):
    from fluidaudio_b200 import _lib
    N = emb.shape[0]
    labels, info = np.zeros(N, np.int32), _lib.ClusterInfo()
    _lib.check(gpu_lib.fa_diarize_cluster(emb.ctypes.data, rho.ctypes.data, N, emb.shape[1], rho.shape[1], psi.ctypes.data,
                                          C.byref(cfg), labels.ctypes.data, None, None, 0, C.byref(info)),
               "fa_diarize_cluster")
    return info


def _default_cfg():
    from fluidaudio_b200 import _lib
    cfg = _lib.ClusterConfig()
    _lib.load().fa_cluster_default_config(C.byref(cfg))
    return cfg


def pipeline_launches(N, info, R, max_it, kmeans=0):
    """cluster_pipeline: widen + finite rows, gather (NaN rows dropped), normalise + AHC (two or more training rows),
    VBx, centroids (or K-Means + centroid normalisation when a speaker-count constraint re-clusters), assignment"""
    Tn, S = info.training_count, info.initial_clusters
    n = 2 + (2 if Tn != N else 0)
    if Tn >= 2:
        n += 1 + ahc_launches(Tn)
    n += vbx_launches(S, R, max_it)
    n += kmeans + 1 if info.was_adjusted else centroid_launches(S)
    return n + 1


@pytest.mark.gpu
def test_diarize_cluster(gpu_lib):
    from fluidaudio_b200 import synth
    emb, _ = synth.speaker_embeddings(120, 256, 4, seed=4)
    rho, psi = synth.synthetic_plda(emb)
    cfg = _default_cfg()
    R, max_it = rho.shape[1], cfg.vbx.max_iterations
    # plain
    d, info = _delta(lambda: _cluster(gpu_lib, emb, rho, psi, cfg))
    assert info.training_count == 120 and info.centroid_count > 0
    assert d == pipeline_launches(120, info, R, max_it), d
    # NaN rows: the finite rows are gathered first
    bad = emb.copy()
    bad[[3, 50, 77]] = np.nan
    d, info = _delta(lambda: _cluster(gpu_lib, bad, rho, psi, cfg))
    assert info.training_count == 117
    assert d == pipeline_launches(120, info, R, max_it), d
    # a single finite row: no AHC
    one = np.full_like(emb[:5], np.nan)
    one[2] = emb[2]
    d, info = _delta(lambda: _cluster(gpu_lib, one, rho[:5].copy(), psi, cfg))
    assert info.training_count == 1 and info.initial_clusters == 1
    assert d == pipeline_launches(5, info, R, max_it), d
    # num_speakers away from what VBx finds: K-Means re-clusters the training rows (the same call as fa_kmeans_cluster)
    target = 7
    cfg_k = _default_cfg()
    cfg_k.num_speakers = target
    d, info = _delta(lambda: _cluster(gpu_lib, emb, rho, psi, cfg_k))
    assert info.was_adjusted == 1 and info.centroid_count == target
    km, _ = _delta(lambda: _kmeans(gpu_lib, emb.astype(np.float64), target, 100, 10))
    assert d == pipeline_launches(120, info, R, max_it, kmeans=km), (d, km)


@pytest.mark.gpu
def test_diarize_cluster_batch(gpu_lib):
    from fluidaudio_b200 import _lib, synth
    emb, _ = synth.speaker_embeddings(900, 256, 4, seed=6)
    rho, psi = synth.synthetic_plda(emb)
    offsets = np.array([0, 250, 600, 900], np.int64)
    cfg = _default_cfg()
    per_set = 0
    for m in range(3):
        a, b = offsets[m], offsets[m + 1]
        per_set += _delta(lambda: _cluster(gpu_lib, emb[a:b].copy(), rho[a:b].copy(), psi, cfg))[0]
    labels = np.zeros(900, np.int32)
    d, _ = _delta(lambda: _lib.check(gpu_lib.fa_diarize_cluster_batch(emb.ctypes.data, rho.ctypes.data, offsets.ctypes.data,
                                                                       3, 256, rho.shape[1], psi.ctypes.data, C.byref(cfg),
                                                                       labels.ctypes.data, None), "batch"))
    assert d == per_set, (d, per_set)
