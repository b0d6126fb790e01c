"""CPU tests of the product's host side (no GPU needed, no compute calls into the CUDA library):

* the C-ABI library loads and exports every symbol the public headers declare;
* argument contracts that are decided before any device work (the reference's own status codes);
* "no CPU fallback": without an H100 every compute entry point fails loudly;
* the product never touches oracle/;
* the device code's per-lane FFT / mel math and the merge kernel's control plane, compiled for the host from the
  SAME headers the kernels use (tests/emul/*.cpp), against the oracle and the reference goldens;
* sharding helpers, including a 2-rank gloo run.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from fluidaudio_b200 import _lib, sharding, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    return _lib.load()


def _declared_functions(header):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(r"\b(fa_[a-z0-9_]+|fastcluster_compute_centroid_linkage)\s*\(", text))


def test_library_exports_every_declared_symbol(lib):
    declared = _declared_functions("fluidaudio_b200.h") | _declared_functions("FastClusterWrapper.h")
    assert "fastcluster_compute_centroid_linkage" in declared and len(declared) >= 35
    out = subprocess.check_output(["nm", "-D", "--defined-only", _lib.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    assert declared <= exported, f"declared but not exported: {sorted(declared - exported)}"
    assert set(_lib.EXPORTED_SYMBOLS) == declared
    # nothing but the C ABI leaks out of the shared object
    assert all(s.startswith("fa_") or s.startswith("fastcluster_") for s in exported), sorted(exported)[:10]


def test_reference_argument_contract_needs_no_device(lib):
    """FastClusterWrapper.cpp:203-223 — these statuses are decided before any clustering work."""
    f = lib.fastcluster_compute_centroid_linkage
    x = np.ones((3, 2))
    z = np.zeros(8)
    assert f(None, 3, 2, z.ctypes.data, 8) == 1
    assert f(x.ctypes.data, 3, 2, None, 8) == 1
    assert f(x.ctypes.data, 0, 2, z.ctypes.data, 8) == 0
    assert f(x.ctypes.data, 3, 0, z.ctypes.data, 8) == 1
    assert f(x.ctypes.data, 2 ** 31, 2, z.ctypes.data, 8) == 2
    assert f(x.ctypes.data, 3, 2 ** 31, z.ctypes.data, 8) == 2
    assert f(x.ctypes.data, 3, 2, z.ctypes.data, 7) == 3
    assert f(x.ctypes.data, 1, 2, z.ctypes.data, 0) == 0
    assert np.all(z == 0)


def test_swift_level_guards_need_no_device(lib):
    from fluidaudio_b200.clustering import AHCClustering
    ahc = AHCClustering()
    assert ahc.cluster([], 0.7).size == 0                                   # AHCClusteringTests.swift:12-15
    assert ahc.cluster(np.zeros((3, 0)), 0.7).tolist() == [0, 0, 0]         # :137-145
    labels = np.zeros(1, np.int32)
    assert lib.fa_ahc_cluster(np.ones((1, 3)).ctypes.data, 1, 3, 0.7, labels.ctypes.data) == 0 and labels[0] == 0


def test_no_cpu_fallback_without_a_device(lib):
    """Run in a child process with every GPU hidden (CUDA_VISIBLE_DEVICES=""), so the behaviour is checked on machines with
    and without one."""
    code = (
        "import sys, numpy as np; sys.path.insert(0, %r)\n"
        "from fluidaudio_b200 import _lib, synth\n"
        "from fluidaudio_b200.mel import AudioMelSpectrogram\n"
        "from fluidaudio_b200.clustering import OfflineClusterer, centroid_linkage\n"
        "assert _lib.device_count() == 0\n"
        "try:\n"
        "    AudioMelSpectrogram(); raise SystemExit('mel ran without a device')\n"
        "except _lib.FluidAudioError as e:\n"
        "    assert e.status == 6 and 'no CPU fallback' in str(e), str(e)\n"
        "emb, _ = synth.speaker_embeddings(50, 16, 2)\n"
        "try:\n"
        "    OfflineClusterer().cluster(emb, emb.astype(np.float64)); raise SystemExit('clustering ran without a device')\n"
        "except _lib.FluidAudioError:\n"
        "    pass\n"
        "st, _ = centroid_linkage(np.eye(3))\n"
        "assert st == 5, st      # the Swift caller maps a non-zero status to identity labels (AHCClustering.swift:52-55)\n"
        "print('NO_DEVICE_OK')\n" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CUDA_VISIBLE_DEVICES=""), capture_output=True,
                         text=True, timeout=300)
    assert "NO_DEVICE_OK" in out.stdout, (out.stdout[-500:], out.stderr[-1500:])


def test_product_never_imports_or_links_the_oracle():
    pkg = os.path.join(ROOT, "fluidaudio_b200")
    for dirpath, _, files in os.walk(pkg):
        for name in files:
            if name.endswith((".py", ".cu", ".cuh", ".h", ".cpp")) or name == "Makefile":
                text = open(os.path.join(dirpath, name), errors="ignore").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f"{name} imports oracle"
                assert "liboracle" not in text and "oracle_" not in text, f"{name} references the oracle"
    out = subprocess.check_output(["ldd", _lib.LIB_PATH], text=True)
    assert "oracle" not in out


def test_helpers_that_run_on_the_host(lib, oracle):
    # sizing calls and argument checks need no device (the arithmetic of these two entry points runs on the GPU:
    # tests/test_gpu_parity.py::test_standalone_normalise_and_linear_resample)
    n = C.c_int64()
    assert lib.fa_linear_resample(None, 1000, 3, 48000.0, 16000.0, None, 0, C.byref(n)) == 0 and n.value == 333
    assert lib.fa_linear_resample(None, 1000, 0, 48000.0, 16000.0, None, 0, C.byref(n)) != 0
    z = np.ones((3, 4), np.float32)
    assert lib.fa_mel_normalize_per_feature(z.ctypes.data, 3, 4, 0) == 0 and not z.any()   # no valid frame: all padding
    assert lib.fa_mel_normalize_per_feature(None, 3, 4, 1) != 0
    from fluidaudio_b200.clustering import dendrogram_cut
    rng = np.random.default_rng(5)
    for n in (2, 7, 40):
        xx = oracle.l2_normalize_rows(rng.standard_normal((n, 3)))
        _, z = oracle.centroid_linkage(xx)
        for thr in (0.0, 0.5, 1.0, 2.5, float("nan")):
            assert np.array_equal(dendrogram_cut(z, n, thr), oracle.dendrogram_cut(z, n, thr))


def test_constrained_assignment_host_functions(lib, oracle):
    """The per-chunk Hungarian matching is host code inside the library (exact integer logic, O(chunks K^3)):
    reference KATs (HungarianAssignmentTests.swift, ConstrainedClusterAssignmentTests.swift) and equality with the
    oracle on tie-heavy random problems."""
    from fluidaudio_b200.clustering import ConstrainedClusterAssignment as Cc, HungarianAssignment as H, \
        build_chunk_assignments
    assert H.solve([4, 1, 3, 2, 0, 5, 3, 2, 2], 3) == [1, 0, 2] and H.solve([1, 2, 0, 10], 2) == [1, 0]
    assert H.solve([], 0) == []
    assert H.max_score_assignment([[0.9, 0.1], [0.8, 0.2]]) == [0, 1]
    assert H.max_score_assignment([[0.1, 0.9, 0.3]]) == [1]
    assert H.max_score_assignment([[0.9], [0.5], [0.7]]) == [0, -1, -1]
    assert H.max_score_assignment([[float("nan"), 0.2], [0.6, 0.5]]) == [1, 0]
    assert H.max_score_assignment([]) == [] and H.max_score_assignment([[], []]) == [-1, -1]
    assert Cc.assign([[0.9, 0.3], [0.8, 0.6]], [0, 0]) == [0, 1]
    assert Cc.assign([[0.9, 0.3], [0.8, 0.6]], [0, 1]) == [0, 0]
    assert Cc.assign([[0.9], [0.2]], [0, 0]) == [0, -2]
    assert Cc.assign([[0.1, 0.7, 0.4], [0.5, 0.2, 0.9]], [3, 7]) == [1, 2]
    assert Cc.assign([], []) == [] and Cc.assign([[0.50, 0.55], [0.10, 0.90]], [0, 0]) == [0, 1]
    rng = np.random.default_rng(0)
    for _ in range(300):
        rows, cols = int(rng.integers(1, 5)), int(rng.integers(1, 7))
        sc = np.round(rng.random((rows, cols)), 2)
        if rng.random() < 0.2:
            sc[rng.integers(rows), rng.integers(cols)] = np.inf if rng.random() < 0.5 else np.nan
        assert H.max_score_assignment(sc.tolist()) == oracle.max_score_assignment(sc).tolist()
    n, k = 700, 5
    sc = np.round(rng.random((n, k)), 3)
    chunk = rng.integers(0, 250, n)
    spk = rng.integers(0, 3, n)
    got = np.array(Cc.assign(sc, chunk), np.int32)
    assert np.array_equal(got, oracle.constrained_assign(sc, chunk))
    assert np.array_equal(build_chunk_assignments(chunk, spk, got, 250, 3, k),
                          oracle.build_chunk_assignments(chunk, spk, got, 250, 3, k))
    for c in np.unique(chunk):          # distinct clusters inside a chunk (or -2)
        a = got[chunk == c]
        assert len(set(a[a >= 0].tolist())) == (a >= 0).sum()


# ------------------------------------------------------------------------------------------------ device code on the host
def _compile(src, out):
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", out,
                           os.path.join(ROOT, "tests", "emul", src)])
    return C.CDLL(out)


def test_kernel_lane_math_matches_oracle(tmp_path, oracle):
    """mel_core.cuh (the per-lane FFT256 / recombination / banded mel / log the CUDA kernel runs) emulated lane by
    lane on the host vs the oracle: same frames, |delta log-mel| <= 1e-4."""
    L = _compile("mel_emul.cpp", str(tmp_path / "libmel_emul.so"))
    f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
    L.mel_emul.argtypes = [f32p, C.c_longlong, C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, f32p,
                           f32p, C.c_float, C.c_int, C.c_longlong, f32p]
    for nm, gen, n in ((80, synth.tone_noise_audio, 16000 * 4 + 137), (128, synth.speech_like_audio, 16000 * 3)):
        a = gen(n)
        ref, T, _ = oracle.mel_flat_transposed(oracle.mel_config(n_mels=nm), a)
        out = np.zeros((T, nm), np.float32)
        assert L.mel_emul(a, a.size, 0.0, 160, 400, 56, 256, np.float32(0.97), nm, oracle.mel_filterbank(512, nm),
                          oracle.hann_window(), np.float32(2.0 ** -24), 0, T, out) == 0
        assert np.abs(out - ref).max() <= 1e-4
    # the float32-pair value type (two frames per warp, FA_MEL_PRECISION_F32) through the same per-lane code: index math of
    # the pair rows, exact-rounded twiddle scalars; float32 transform noise stays inside the bar on these fixtures
    L.mel_emul_f32x2.argtypes = L.mel_emul.argtypes
    for nm, gen, n in ((80, synth.tone_noise_audio, 16000 * 4 + 137), (128, synth.speech_like_audio, 16000 * 3)):
        a = gen(n)
        ref, T, _ = oracle.mel_flat_transposed(oracle.mel_config(n_mels=nm), a)
        out = np.zeros((T, nm), np.float32)
        assert L.mel_emul_f32x2(a, a.size, 0.0, 160, 400, 56, 256, np.float32(0.97), nm, oracle.mel_filterbank(512, nm),
                                oracle.hann_window(), np.float32(2.0 ** -24), 0, T, out) == 0
        assert np.abs(out - ref).max() <= 1e-4
    # legacy compute(): window at offset 0, no padding, no pre-emphasis
    a = synth.tone_noise_audio(8000)
    ref, T = oracle.mel_legacy(oracle.mel_config(n_mels=80), a)
    out = np.zeros((T, 80), np.float32)
    assert L.mel_emul(a, a.size, 0.0, 160, 400, 0, 0, np.float32(0.0), 80, oracle.mel_filterbank(512, 80),
                      oracle.hann_window(), np.float32(2.0 ** -24), 0, T, out) == 0
    assert np.abs(out.T - ref).max() <= 1e-4

    # The configuration space of the specialised kernel: even hops, window lengths on both sides of the mid_full boundary
    # (buffer positions [64, 448)) centred and at offset 0, mel counts with empty filters, other sample rates, every log
    # floor (subnormal and zero too) in both floor modes, with and without pre-emphasis.  FP64 transform: DESIGN's bar,
    # |d| <= 1e-5 + 4e-7 |ref| (the second term: 2 ulp of the log at large magnitudes); float32 pairs: 1e-4 (f32_bar).
    hops = (2, 64, 128, 158, 256, 320, 512, 514, 1000)
    wins = (512, 449, 448, 400, 385, 384, 383, 256, 64)
    mels = (1, 3, 23, 40, 81, 128, 200, 257)
    rates = (8000, 22050, 48000, 16000)
    floors = (2.0 ** -24, 1e-10, 1e-38, 0.0)
    worst = {"f64": 0.0, "f32x2": 0.0}

    def run(fn, x, cfg, mode, last, off, nm, sr):
        """One emulator call against the oracle in the same mode: returns (emulated, oracle) as [T x nMels]."""
        if mode == 2:
            ref, T = oracle.mel_legacy(cfg, x)
            ref = ref.T
        else:
            ref, T, _ = oracle.mel_flat_transposed(cfg, x, last=last, padding_mode=mode)
            ref = ref[:T]
        out = np.zeros((T, nm), np.float32)
        pad, pre = (256 if mode == 0 else 0), (np.float32(0.0) if mode == 2 else np.float32(cfg.preemph))
        assert fn(x, x.size, last, cfg.hop_length, cfg.win_length, off, pad, pre, nm, oracle.mel_filterbank(512, nm, sr),
                  oracle.hann_window(cfg.win_length), np.float32(cfg.log_floor), cfg.log_floor_mode, T, out) == 0
        return out, ref

    def check(out, ref, fb, bar, what):
        """NaN frames of the oracle (dense filterbank: every mel) must be NaN in every non-empty band; elsewhere the values
        agree within the bar, non-finite values (log 0 = -inf) exactly."""
        nan_rows = np.isnan(ref).all(axis=1)
        assert not np.isnan(ref[~nan_rows]).any(), what
        band = fb.any(axis=1)
        assert np.isnan(out[nan_rows][:, band]).all(), what
        o, r = out[~nan_rows], ref[~nan_rows]
        fin = np.isfinite(r)
        assert np.array_equal(o[~fin], r[~fin]) and np.isfinite(o[fin]).all(), what
        top = np.broadcast_to(np.where(np.isfinite(r), r, -np.inf).max(axis=1, keepdims=True), r.shape)
        d = np.abs(o[fin] - r[fin])
        ok = d <= bar(r[fin], top[fin])
        assert ok.all(), (what, float(d.max()), "largest so far", worst)
        return float(d.max()) if d.size else 0.0, nan_rows

    fp64_bar = lambda r, top: 1e-5 + 4e-7 * np.abs(r)
    # float32 pairs: 1e-4, except for mel values more than 12 nats below the frame's strongest one.  There the float32
    # transform's rounding noise (a fraction of an ulp of the strongest line in every bin, DESIGN §2) dominates the value:
    # near-DC bands after pre-emphasis at 22.05 / 48 kHz reach 3e-4 at 18 nats down; the bar grows with exp(depth), capped
    # at 2e-3 (the largest deviation measured here is 5.1e-4, on the GPU over tests/test_gpu_mel_sweep.py 9.8e-4).
    f32_bar = lambda r, top: np.minimum(2e-3, 1e-4 * np.maximum(1.0, np.exp(top - r - 12.0)))
    i = 0
    for hop in hops:
        for win in wins:
            for mode in (0, 1, 2):   # centred with and without the centre padding; legacy: offset 0, no pre-emphasis
                nm, sr, fl = mels[i % len(mels)], rates[i % len(rates)], floors[i % len(floors)]
                clamped, pre = (i // len(floors)) % 2, (0.97 if (i // 2) % 2 == 0 else 0.0)
                i += 1
                cfg = oracle.mel_config(sample_rate=sr, n_mels=nm, hop_length=hop, win_length=win, preemph=pre,
                                        log_floor=fl, log_floor_mode=clamped)
                off = 0 if mode == 2 else (512 - win) // 2
                frames = (17, 33, 2, 16, 1, 31, 15)[i % 7]
                x = synth.tone_noise_audio(max(1, (frames - 1) * hop + 512 - (256 if mode == 0 else 0)), seed=i)
                fb = oracle.mel_filterbank(512, nm, sr)
                what = dict(hop=hop, win=win, mode=mode, n_mels=nm, sr=sr, floor=fl, clamped=clamped, pre=pre)
                out, ref = run(L.mel_emul, x, cfg, mode, 0.3, off, nm, sr)
                worst["f64"] = max(worst["f64"], check(out, ref, fb, fp64_bar, what)[0])
                out, ref = run(L.mel_emul_f32x2, x, cfg, mode, 0.3, off, nm, sr)
                worst["f32x2"] = max(worst["f32x2"], check(out, ref, fb, f32_bar, what)[0])
    assert i == len(hops) * len(wins) * 3

    # NaN samples: at the first and last in-window sample of a frame (the frame must be NaN), and one sample outside the
    # window on either side (the kernel must select the in-window samples, not multiply the whole buffer by a window that is
    # zero there: NaN * 0 = NaN).  Every window placement, both floor modes, both value types.
    for win in wins:
        for mode in (0, 2):
            for clamped in (0, 1):
                nm, hop = 40, 160
                cfg = oracle.mel_config(n_mels=nm, hop_length=hop, win_length=win, preemph=0.97, log_floor=1e-10,
                                        log_floor_mode=clamped)
                off, pad = (0, 0) if mode == 2 else ((512 - win) // 2, 256)
                f = 6
                for j, inside in ((off, True), (off + win - 1, True), (off - 1, False), (off + win, False)):
                    if j < 0 or j >= 512:
                        continue
                    x = synth.tone_noise_audio(16 * hop + 512, seed=win + j)
                    x[f * hop + j - pad] = np.nan
                    for fn, bar in ((L.mel_emul, fp64_bar), (L.mel_emul_f32x2, f32_bar)):
                        what = dict(win=win, mode=mode, clamped=clamped, j=j, fn=fn.__name__)
                        out, ref = run(fn, x, cfg, mode, 0.0, off, nm, 16000)
                        _, nan_rows = check(out, ref, oracle.mel_filterbank(512, nm), bar, what)
                        # not vacuous: a NaN inside the window poisons the frame, one outside it (after pre-emphasis
                        # on the right; on the left only without it) leaves the frame finite
                        if inside:
                            assert nan_rows[f], what
                        elif j > off or mode == 2:
                            assert not nan_rows[f] and np.isfinite(out[f]).all(), what
    print("largest |d log-mel| vs the oracle:", worst)


def test_sinc_kernel_index_math_is_exact(tmp_path, oracle):
    """resample_core.cuh (the per-CTA and per-thread index arithmetic of sinc_kernel) on the host: for the extreme ratios
    make_design accepts, every thread of CTAs at the start, the middle (aligned and not: the fused pipeline launches at any
    output) and the end of an hour-long output gets n0 = floor(i M / L) and phase (i M) mod L exactly, in the index width
    the kernel selects; the staged span covers every tap any thread reads and fits the shared memory the launch asks for.
    32-bit offsets are shown to be wrong where the kernel must not select them (44100.001 Hz: L = 16e6, M = 44 100 001)."""
    L_ = _compile("resample_emul.cpp", str(tmp_path / "libresample_emul.so"))
    i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
    L_.resample_index.argtypes = [C.c_longlong, C.c_longlong, C.c_int, C.c_longlong, C.c_int, C.c_int, i64p, i64p, i64p,
                                  i64p]
    L_.resample_narrow.argtypes = [C.c_longlong, C.c_longlong]
    L_.resample_smem_floats.argtypes = [C.c_longlong, C.c_longlong, C.c_int]
    L_.resample_smem_floats.restype = C.c_longlong

    def run(d, i0, count, wide):
        n0, ph, dn, span = (np.zeros(count, np.int64), np.zeros(count, np.int64), np.zeros(count, np.int64),
                            np.zeros(1, np.int64))
        assert L_.resample_index(d.L, d.M, d.half, i0, count, int(wide), n0, ph, dn, span) == 0
        return n0, ph, dn, int(span[0])

    def exact(d, i0, count):
        return ([(i0 + j) * d.M // d.L for j in range(count)], [(i0 + j) * d.M % d.L for j in range(count)])

    down = 1                    # the largest decimation ratio make_design accepts (window bound); upsampling keeps H = 24
    while True:
        try:
            oracle.sinc_design(16000 * (down + 1), 16000)
        except ValueError:
            break
        down += 1
    assert down == 168
    pairs = [(16000 * down, 16000), (16000 * down - 0.001, 16000), (1000, 4000000.001), (44100, 16000), (44100.5, 16000),
             (44100.001, 16000), (48000.001, 16000), (47999.998, 16000), (16001, 16000), (8000.1, 16000),
             (16000, 192000.001), (4000000.003, 4000000.001)]
    selected = {}
    for rin, rout in pairs:
        d = oracle.sinc_design(rin, rout)
        wide = not L_.resample_narrow(d.L, d.M)
        selected[(rin, rout)] = "64" if wide else "32"
        assert wide == (255 * d.M + d.L >= 2 ** 32)
        taps, smem = 2 * d.half, L_.resample_smem_floats(d.L, d.M, 2 * d.half)
        count = oracle.resample_output_count(int(round(rin * 3600)), rin, rout)
        mid = count // 2 // 256 * 256
        for i0, n in ((0, 256), (mid, 256), (mid + 77, 256), ((count - 1) // 256 * 256, count - (count - 1) // 256 * 256)):
            n0, ph, dn, span = run(d, i0, n, wide)
            e_n0, e_ph = exact(d, i0, n)
            assert n0.tolist() == e_n0 and ph.tolist() == e_ph, (rin, rout, i0)
            assert dn[0] == 0 and (dn + taps).max() <= span <= smem, (rin, rout, i0, span, smem)
    # the parent's 32-bit arithmetic at 44100.001 Hz: most threads of a CTA read the wrong window at the wrong phase
    d = oracle.sinc_design(44100.001, 16000)
    n0, ph, _, _ = run(d, 256 * 1000, 256, False)
    e_n0, e_ph = exact(d, 256 * 1000, 256)
    assert (n0 != np.array(e_n0)).sum() > 100 and selected[(44100.001, 16000)] == "64"
    assert selected[(44100, 16000)] == selected[(16000 * down, 16000)] == selected[(16000, 192000.001)] == "32"
    # i0 * M passes 2^63 within the hour at 4 MHz: the split form keeps n0 exact (checked above)
    assert (count - 1) * 4000000003 >= 2 ** 63


def test_merge_control_plane_matches_reference_goldens(tmp_path, golden_dir, oracle):
    """ahc_core.cuh (slot-indexed heap + live bitmap, the code the device master warp runs) driven on the host in the
    merge kernel's order: dendrograms must equal the reference's bit for bit."""
    L = _compile("ahc_emul.cpp", str(tmp_path / "libahc_emul.so"))
    g = np.load(os.path.join(golden_dir, "ahc_reference.npz"))
    for name in sorted({k.rsplit("__", 1)[0] for k in g.files}):
        x = np.ascontiguousarray(g[name + "__x"])
        z = np.zeros((x.shape[0] - 1, 4))
        assert L.ahc_emul(x.ctypes.data_as(C.c_void_p), x.shape[0], x.shape[1], z.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(z, g[name + "__z"]), name
    rng = np.random.default_rng(17)
    for n, d in ((300, 8), (257, 3)):
        x = np.round(rng.standard_normal((n, d)), 1)          # coarse grid: many exactly tied distances
        z = np.zeros((n - 1, 4))
        assert L.ahc_emul(x.ctypes.data_as(C.c_void_p), n, d, z.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(z, oracle.centroid_linkage(x)[1])
    bad = rng.standard_normal((10, 3)); bad[4, 1] = np.nan
    assert L.ahc_emul(bad.ctypes.data_as(C.c_void_p), 10, 3, np.zeros((9, 4)).ctypes.data_as(C.c_void_p)) == 5


PLACEMENT_FIELDS = ("status", "level", "idx16", "cap_slots", "resident", "workers", "slots_per_cta", "rounds", "capacity",
                    "smem", "filter", "keep_tmin", "filter_rows")


@pytest.fixture(scope="module")
def placement_lib(tmp_path_factory):
    """ahc_placement.h compiled on the host, and the GPU sweep's restatement of it"""
    import importlib.util
    L = _compile("ahc_placement_emul.cpp", str(tmp_path_factory.mktemp("placement") / "libahc_placement.so"))
    spec = importlib.util.spec_from_file_location("ahc_sweep", os.path.join(ROOT, "tests", "test_gpu_ahc_sweep.py"))
    sweep = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sweep)

    def plan(N, D, W, force_global=False, force_stream=False, filter_min_n=2048):
        out = (C.c_longlong * 13)()
        L.ahc_placement(N, D, W, int(force_global), int(force_stream), filter_min_n, out)
        return dict(zip(PLACEMENT_FIELDS, out))

    def lanes(set_count, n_max, D, sms):
        out = (C.c_int * 2)()
        L.ahc_batch_lanes(set_count, C.c_longlong(n_max), D, sms, out)
        return tuple(out)

    return plan, lanes, sweep


def test_merge_kernel_placement_boundaries(placement_lib):
    """plan_linkage at every boundary of the placement table (DESIGN.md section 4.2), for a 132-SM H100 SXM (131
    worker CTAs) and a 114-SM H100 PCIe (113)."""
    plan, _, sweep = placement_lib
    for W in (131, 113):
        # master state in shared memory: level 3 (heap + nn + node_of), 2 (heap + nn), 1 (heap), 0 (global)
        for N, level in ((11376, 3), (11377, 2), (14176, 2), (14177, 1), (18808, 1), (18809, 0), (65535, 0)):
            p = plan(N, 4, W)
            assert (p["level"], p["idx16"]) == (level, int(level > 0)), (W, N, p)
        assert plan(1500, 4, W, force_global=True)["level"] == 0
        # node vectors per worker CTA, and the resident -> streamed flip at cap(D) * W
        for D, cap in ((1, 128), (219, 128), (220, 127), (256, 109), (512, 53), (1024, 25), (1536, 15), (2048, 11),
                       (4096, 4), (7196, 1), (7197, 0)):
            assert plan(4, D, W)["cap_slots"] == cap, (D, cap)
            if cap:
                assert plan(cap * W, D, W)["resident"] == 1 and plan(cap * W + 1, D, W)["resident"] == 0, (W, D)
                assert plan(cap * W, D, W, force_stream=True)["resident"] == 0
            else:
                assert plan(4, D, W)["status"] == 5                         # D >= 7 197: FA_RUNTIME_ERROR
        assert plan(min(16768, 128 * W), 4, W)["smem"] <= 227 * 1024 - 2048
        # streamed rounds: 2 from 128 W + 1, 16 at the capacity W * 2 048, refused one point past it
        assert plan(128 * W + 1, 4, W)["rounds"] == 2
        assert plan(256 * W + 1, 4, W)["rounds"] == 3
        top = plan(W * 2048, 1, W)
        assert (top["status"], top["rounds"], top["workers"], top["capacity"]) == (0, 16, W, W * 2048)
        assert plan(W * 2048 + 1, 1, W)["status"] == 5 and plan(W * 2048 + 1, 4096, W)["status"] == 5
        # float32 filter from N = 2 048; its pass 2 is the rows kernel while the bounds are kept and D <= 1 536
        assert plan(2047, 16, W)["filter"] == 0 and plan(2048, 16, W)["filter"] == 1
        assert plan(2048, 16, W, filter_min_n=0)["filter"] == 0 and plan(3, 16, W, filter_min_n=2)["filter"] == 1
        assert plan(32768, 4, W)["keep_tmin"] == 1 and plan(32769, 4, W)["keep_tmin"] == 0
        assert plan(32768, 4, W)["filter_rows"] == 1 and plan(32769, 4, W)["filter_rows"] == 0
        assert plan(2048, 1536, W)["filter_rows"] == 1 and plan(2048, 1537, W)["filter_rows"] == 0
    # the sweep's formulas for a 132-SM device are these numbers
    assert sweep.level_limits() == [11376, 14176, 18808] and sweep.d_limit() == 7196


def test_merge_kernel_placement_restatement_is_exact(placement_lib):
    """The GPU sweep computes its shapes from a Python restatement of ahc_placement.h: it must agree field for field."""
    plan, lanes, sweep = placement_lib
    rng = np.random.default_rng(3)
    Ns = {2, 3, 31, 32, 33, 2047, 2048, 11376, 11377, 14176, 14177, 14279, 14280, 16637, 16638, 16768, 16769, 18808,
          18809, 32768, 32769, 33537, 65535, 65536, 65537, 231424, 231425, 268288, 268289, 300000}
    Ns |= set(rng.integers(2, 300000, 40).tolist())
    Ds = {1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 33, 219, 220, 256, 1023, 1024, 1536, 1537, 2048, 4096, 7196, 7197, 9000}
    for W in (1, 2, 32, 43, 65, 113, 131):
        for N in sorted(Ns):
            for D in sorted(Ds):
                for hooks in ({}, {"force_global": True, "force_stream": True}, {"filter_min_n": 0}):
                    want = plan(N, D, W, **hooks)
                    assert sweep.placement(N, D, W, **hooks) == want, (N, D, W, hooks, want)
    for sms in (8, 66, 114, 132):
        for count in (1, 2, 3, 4, 7):
            for n_max in sorted(Ns):
                for D in (4, 256, 2048, 7197):
                    assert sweep.batch_lanes(count, n_max, D, sms) == lanes(count, n_max, D, sms), (sms, count, n_max, D)


def test_batch_lanes_keep_every_set_within_its_lane(placement_lib):
    """fa_diarize_cluster_batch runs sets side by side in lanes of SMs / lanes - 1 worker CTAs.  Whatever lane count
    the rule picks, a set the single call accepts must fit its lane's streamed capacity; otherwise the lane's linkage
    fails and the pipeline turns that set into identity labels (a 65 537-row set among four on 132 SMs: 32 workers hold
    65 536 slots)."""
    plan, lanes, _ = placement_lib
    for sms in (132, 114, 66, 8):
        W = sms - 1
        sizes = {2, 300, 5000, 14279, 14280, 16768, 16769, 65536, 65537, 88064, 88065, 133120, 133121, W * 2048 - 31,
                 W * 2048, W * 2048 + 1}
        for D in (1, 4, 220, 256, 1024, 2048, 7196, 7197):
            for n_max in sorted(sizes):
                single = plan(n_max, D, W)["status"]
                for count in range(1, 7):
                    n_lanes, limit = lanes(count, n_max, D, sms)
                    assert 1 <= n_lanes <= min(count, 4) and (limit == 0) == (n_lanes == 1)
                    lane = plan(n_max, D, min(W, limit) if limit else W)
                    assert lane["status"] == single, (sms, D, n_max, count, n_lanes, limit)
    assert lanes(4, 65537, 4, 132) == (3, 43) and lanes(4, 20000, 4, 132) == (4, 32) and lanes(4, 5000, 256, 132)[0] == 2
    assert lanes(4, 132 * 2048, 4, 132) == (1, 0)


# ------------------------------------------------------------------------------------------------ sharding
def test_float32_filter_bound_is_rigorous():
    """The AHC initial pass trusts E_ij = c1 r_i r_j + c2 (n_i + n_j), c1 = 2.02 (D + 3) 2^-24, c2 = 2e-12
    (ahc_kernels.cu: ahc_filter_prep / tile128 / rows) to bracket the reference's sequential double chain from a float32
    inner product of float32-converted inputs, and evaluates the bracket in float32 interval arithmetic.  Restated here in
    numpy (directed rounding through nextafter) and checked on inputs chosen to stress it: unit rows, near-duplicates,
    exact duplicates, rows of very different norm, widths that are not multiples of eight, float32 sums in three orders."""
    rng = np.random.default_rng(7)
    f32, f64 = np.float32, np.float64

    def chain(a, b):                      # fastcluster's sq. distance: sum += (a_k - b_k)^2, every operation rounded
        s = f64(0.0)
        for k in range(a.size):
            d = f64(a[k] - b[k])
            s = f64(s + f64(d * d))
        return s

    def rd(x):                            # float64 -> float32 rounded down / up
        y = f32(x)
        return y if f64(y) <= x else np.nextafter(y, f32(-np.inf))

    def ru(x):
        y = f32(x)
        return y if f64(y) >= x else np.nextafter(y, f32(np.inf))

    worst = 0.0
    for D in (256, 255, 64, 13):
        c1 = 2.02 * (D + 3) * 2.0 ** -24
        c2 = 2e-12
        base = rng.standard_normal((24, D))
        base /= np.linalg.norm(base, axis=1, keepdims=True)
        rows = [base[i] for i in range(24)]
        rows += [base[0] + 1e-7 * rng.standard_normal(D), base[1] * (1 + 1e-9), base[2].copy(), base[3] * 37.5, base[4] * 1e-3,
                 np.round(base[5] * 4) / 4, np.zeros(D)]
        X = np.asarray(rows, f64)
        Xf = X.astype(f32)
        n = (X * X).sum(axis=1)                                   # |x|^2 in double (k ascending in the kernel; any order here)
        r = np.array([ru(np.sqrt(v)) * f32(1.000001) for v in n], f32)
        for i in range(len(rows)):
            for j in range(i):
                exact = chain(X[i], X[j])
                dots = (np.dot(Xf[i], Xf[j]),                                          # library order
                        f32(sum(f32(Xf[i][k] * Xf[j][k]) for k in range(D))),          # sequential, products rounded
                        f32(np.sum((Xf[i][::-1] * Xf[j][::-1]).astype(f32), dtype=f32)))   # reversed
                for dot in dots:
                    dot = f64(dot)
                    approx = (n[i] + n[j]) - 2.0 * dot
                    E = c1 * f64(r[i]) * f64(r[j]) + c2 * (n[i] + n[j])
                    assert approx - E <= exact <= approx + E, (D, i, j)
                    if E > 0:
                        worst = max(worst, abs(approx - exact) / E)
                    # the float32 interval form of the tile kernel's epilogue brackets the same bounds
                    s_lo, s_hi = rd(f64(rd(n[i])) + f64(rd(n[j]))), ru(f64(ru(n[i])) + f64(ru(n[j])))
                    e_up = ru(f64(ru(f64(ru(c1)) * f64(r[i]))) * f64(r[j]) + f64(ru(f64(ru(c2)) * f64(s_hi))))
                    hi = ru(f64(ru(-2.0 * dot + f64(s_hi))) + f64(e_up))
                    lo = rd(f64(rd(-2.0 * dot + f64(s_lo))) - f64(e_up))
                    assert f64(lo) <= approx - E + 1e-300 or f64(lo) <= exact
                    assert f64(lo) <= exact <= f64(hi), (D, i, j)
    assert 0.0 < worst < 0.9, worst     # observed error stays below 90 % of the bound (and the check is not vacuous)


def test_sharding_partitions():
    for count, world in ((512, 8), (64, 8), (10, 4), (3, 8), (0, 2)):
        seen = []
        for r in range(world):
            seen += list(sharding.contiguous_shard(count, r, world))
        assert seen == list(range(count))
        sizes = [len(sharding.contiguous_shard(count, r, world)) for r in range(world)]
        assert max(sizes) - min(sizes) <= 1
    costs = [sharding.ahc_cost(n) for n in (5000, 100, 3000, 3000, 800, 4500, 50, 2000)]
    parts = sharding.lpt_partition(costs, 3)
    assert sorted(sum(parts, [])) == list(range(8))
    loads = [sum(costs[i] for i in p) for p in parts]
    assert max(loads) <= 1.34 * sum(costs) / 3          # LPT bound (4/3 - 1/3m) on the makespan
    assert sharding.lpt_partition(costs, 3) == parts    # deterministic


_WORKER = r"""
import os, sys, numpy as np
sys.path.insert(0, {root!r})
from fluidaudio_b200 import sharding
d = sharding.init_distributed("gloo")
mine = sharding.contiguous_shard(10, d.rank, d.world)
labels = np.array([100 * d.rank + i for i in mine], np.int32)
sharding.barrier(d)
mx = sharding.all_reduce_max(d, 1.5 + d.rank)
sm = sharding.all_reduce_sum(d, len(mine))
got = sharding.gather_labels(d, labels, [len(sharding.contiguous_shard(10, r, d.world)) for r in range(d.world)])
import hashlib
digests = np.stack([np.frombuffer(hashlib.sha256(bytes([i])).digest(), np.uint8) for i in mine])
allh = sharding.gather_bytes(d, digests, [len(sharding.contiguous_shard(10, r, d.world)) for r in range(d.world)])
# the C5 plan: 64 equal meetings over the ranks by LPT, labels come back in partition order
parts = sharding.lpt_partition([sharding.ahc_cost(5000)] * 64, d.world)
mine5 = np.concatenate([np.full(3, m, np.int32) for m in parts[d.rank]])
got5 = sharding.gather_labels(d, mine5, [3 * len(p) for p in parts])
if d.is_root:
    assert mx == 2.5 and sm == 10.0, (mx, sm)
    assert got.tolist() == [0, 1, 2, 3, 4, 105, 106, 107, 108, 109], got.tolist()
    assert allh.shape == (10, 32) and all(allh[i].tobytes() == hashlib.sha256(bytes([i])).digest() for i in range(10))
    assert sorted(sum(parts, [])) == list(range(64)) and all(len(p) == 32 for p in parts)
    assert got5.tolist() == [m for p in parts for m in p for _ in range(3)]
    print("GLOO_OK")
sharding.finalize(d)
"""


def test_two_rank_gloo_plumbing(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(root=ROOT))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29533")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", "29533", str(script)],
                         env=env, capture_output=True, text=True, timeout=240)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "GLOO_OK" in out.stdout


# ---- embedding-export files (OfflineDiarizerManager.exportEmbeddings, :913-955): host-only code of the library ----
def _random_export(n, seed=0, e=256, r=128):
    from fluidaudio_b200.export_io import EmbeddingExport
    rng = np.random.default_rng(seed)
    return EmbeddingExport(
        chunk_index=np.sort(rng.integers(0, max(1, n // 2), n)).astype(np.int32),
        speaker_index=rng.integers(0, 3, n).astype(np.int32),
        start_frame=rng.integers(0, 500, n).astype(np.int32), end_frame=rng.integers(500, 1000, n).astype(np.int32),
        start_time=rng.random(n) * 1e3, end_time=rng.random(n) * 1e3 + 1e3,
        embedding256=(rng.standard_normal((n, e)) * 10.0 ** rng.integers(-6, 3, (n, e))).astype(np.float32),
        rho128=rng.standard_normal((n, r)) * 10.0 ** rng.integers(-12, 6, (n, r)),
        cluster=rng.integers(-1, 5, n).astype(np.int32))


def test_embedding_export_round_trip_is_bit_exact(lib, tmp_path):
    from fluidaudio_b200.export_io import EmbeddingExport, PreparedDiarization
    for n in (0, 1, 37):
        ex = _random_export(n, seed=n)
        p = tmp_path / f"export_{n}.json"
        ex.write(p)
        back = EmbeddingExport.read(p)
        assert back.count == n
        for f in ("chunk_index", "speaker_index", "start_frame", "end_frame", "cluster"):
            assert np.array_equal(getattr(back, f), getattr(ex, f))
        for f in ("start_time", "end_time", "embedding256", "rho128"):            # bit patterns, not just values
            a, b = getattr(back, f), getattr(ex, f)
            assert a.dtype == b.dtype and a.tobytes() == b.tobytes()
        if n:
            import json                                                              # the file is plain JSON
            doc = json.load(open(p))
            assert len(doc) == n and set(doc[0]) == {"chunkIndex", "speakerIndex", "startFrame", "endFrame", "startTime",
                                                      "endTime", "embedding256", "rho128", "cluster"}
            prep = PreparedDiarization.load(p)
            assert prep.embedding_count == n and prep.segmentation_chunk_count == int(ex.chunk_index.max()) + 1


def test_embedding_export_reads_foundation_style_json(lib, tmp_path):
    """Key order, whitespace, exponents and unknown keys as Foundation's JSONEncoder / other tools may produce."""
    from fluidaudio_b200.export_io import EmbeddingExport
    text = """ [ {"rho128":[1e-05, -3.5E+2 ,0.1], "cluster" : 2, "embedding256":[0.100000001,-7,1.17549435e-38],
                  "endTime":12.5,"startTime":2,"endFrame":40,"startFrame":4,"speakerIndex":1,"chunkIndex":3,
                  "frameWeights":[0.5,{"nested":[1,2,{"x":null}]},"s\\"tr"], "extra": true },
                 {"chunkIndex":4,"speakerIndex":0,"startFrame":5,"endFrame":6,"startTime":0.25,"endTime":0.5,
                  "embedding256":[1,2,3],"rho128":[4,5,6]} ]\n"""
    p = tmp_path / "swift.json"
    p.write_text(text)
    ex = EmbeddingExport.read(p)
    assert ex.count == 2 and ex.embedding256.shape == (2, 3) and ex.rho128.shape == (2, 3)
    assert ex.chunk_index.tolist() == [3, 4] and ex.speaker_index.tolist() == [1, 0]
    assert ex.start_frame.tolist() == [4, 5] and ex.end_frame.tolist() == [40, 6]
    assert ex.start_time.tolist() == [2.0, 0.25] and ex.end_time.tolist() == [12.5, 0.5]
    assert ex.cluster.tolist() == [2, -1]                                           # absent -> -1, as the writer's default
    assert ex.embedding256[0].tolist() == [np.float32(0.1), -7.0, np.float32(1.17549435e-38)]
    assert ex.rho128[0].tolist() == [1e-05, -350.0, 0.1]


def test_embedding_export_errors_are_reported(lib, tmp_path):
    from fluidaudio_b200.export_io import EmbeddingExport
    with pytest.raises(_lib.FluidAudioError) as e:
        EmbeddingExport.read(tmp_path / "missing.json")
    assert e.value.status == 1 and "cannot open" in str(e.value)
    for name, text, what in (("trunc", '[{"chunkIndex":1,"embedding256":[1,2', "expected"),
                             ("ragged", '[{"embedding256":[1,2],"rho128":[1]},{"embedding256":[1],"rho128":[1]}]', "different"),
                             ("notarray", '{"chunkIndex":1}', "expected '['"),
                             ("frac", '[{"chunkIndex":1.5,"embedding256":[],"rho128":[]}]', "integer"),
                             ("tail", '[] x', "trailing")):
        p = tmp_path / f"{name}.json"
        p.write_text(text)
        with pytest.raises(_lib.FluidAudioError) as e:
            EmbeddingExport.read(p)
        assert e.value.status == 1 and what in str(e.value), (name, str(e.value))


def test_same_partition_helper():
    from fluidaudio_b200.export_io import same_partition
    assert same_partition([0, 0, 1, 2, -2], [5, 5, 3, 9, -1])
    assert not same_partition([0, 0, 1], [1, 2, 2])
    assert not same_partition([0, 1], [0, 0])
    assert not same_partition([0, -2], [0, 1])
    assert not same_partition([0, 1], [0, 1, 2])


def test_speaker_constraints_host_function(lib, oracle):
    """fa_speaker_constraints_resolve needs no device; same table as SpeakerCountConstraintsTests.swift."""
    from fluidaudio_b200.clustering import OfflineDiarizerConfig, SpeakerCountConstraints
    cases = [(100, None, None, None), (100, 3, 1, 10), (5, None, 2, 20), (100, None, 10, 5), (100, 0, None, None),
             (100, -5, None, None), (100, None, 0, 5), (100, None, -3, 5), (1, None, None, None), (7, -1, None, None)]
    for n, num, lo, hi in cases:
        got = SpeakerCountConstraints.resolve(n, num, lo, hi)
        assert (got.min_speakers, got.max_speakers) == oracle.speaker_constraints(n, num, lo, hi)
    c = SpeakerCountConstraints.resolve(100, None, 5, 10)
    assert c.needs_adjustment(3) and c.target_count(3) == 5 and c.num_speakers is None    # :104-113
    c = SpeakerCountConstraints.resolve(100, None, 2, 5)
    assert c.needs_adjustment(8) and c.target_count(8) == 5                               # :115-124
    assert not c.needs_adjustment(3) and c.target_count(3) == 3                           # :126-135
    assert SpeakerCountConstraints.resolve(100, 3, 1, 10).num_speakers == 3
    cfg = OfflineDiarizerConfig().with_speakers(min=2, max=4)
    cc = cfg._c_cluster()
    assert (cc.num_speakers, cc.min_speakers, cc.max_speakers) == (_lib.NO_VALUE, 2, 4)
    cc = cfg.with_speakers(exactly=3)._c_cluster()
    assert (cc.num_speakers, cc.min_speakers, cc.max_speakers) == (3, _lib.NO_VALUE, _lib.NO_VALUE)


def test_headers_are_plain_c_and_link(lib, tmp_path):
    """include/*.h compile as C11 with -Wall -Wextra -pedantic -Werror, and a C program linked against the shared
    library runs the host-only part of the ABI (no GPU needed)."""
    exe = tmp_path / "abi_smoke"
    libdir = os.path.dirname(_lib.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "c", "abi_smoke.c"), "-o", str(exe), "-L", libdir,
                           "-lfluidaudio_b200", f"-Wl,-rpath,{libdir}"])
    out = subprocess.check_output([str(exe)], text=True)
    assert out.startswith("abi ok:")


# ---- timeline reconstruction (OfflineReconstruction.buildSegments): host code of the library vs the oracle -----------
def _synthetic_segmentation(rng, chunks, frames=60, speakers=3, step=20, dur=0.05, k=3):
    """Sliding windows over a piecewise-constant speaker timeline: weights in {~0, ~1}, local slots permuted per chunk."""
    total = step * (chunks - 1) + frames
    truth = np.zeros((total, k), np.float32)
    t = 0
    while t < total:
        length = int(rng.integers(5, 40))
        who = rng.choice(k, size=int(rng.integers(0, 3)), replace=False)
        truth[t:t + length, who] = 1.0
        t += length
    w = np.zeros((chunks, frames, speakers), np.float32)
    hard = np.full((chunks, speakers), -2, np.int32)
    for c in range(chunks):
        perm = rng.permutation(k)[:speakers]
        seg = truth[c * step:c * step + frames]
        for s, cl in enumerate(perm):
            if seg[:, cl].any():
                hard[c, s] = cl
                w[c, :, s] = np.clip(seg[:, cl] * rng.uniform(0.7, 1.0) + rng.uniform(0, 0.05, frames), 0, 1)
    offsets = np.arange(chunks) * step * dur
    return w, hard, offsets, dur, truth


def test_timeline_reconstruction_matches_oracle(lib, oracle):
    from fluidaudio_b200.clustering import OfflineReconstruction
    rng = np.random.default_rng(4)
    for case in range(12):
        chunks = int(rng.integers(1, 30))
        w, hard, offsets, dur, truth = _synthetic_segmentation(rng, chunks)
        kw = dict(min_gap_duration=float(rng.choice([0.0, 0.1, 0.5])), min_segment_duration=float(rng.choice([0.0, 0.2, 1.0])),
                  exclusive_segments=bool(rng.integers(0, 2)))
        use_off = offsets if case % 3 else offsets[: max(1, chunks // 2)]        # missing offsets -> chunk * windowDuration
        got = OfflineReconstruction(dur, window_duration=1.0, **kw).build_segments(w, hard, 3, use_off)
        ref = oracle.build_segments(w, hard, 3, dur, use_off, window_duration=1.0, **kw)
        assert [(s.cluster, s.start_time_seconds, s.end_time_seconds, s.quality_score) for s in got] == \
            [(c, float(a), float(b), float(q)) for c, a, b, q in ref], case
        starts = [s.start_time_seconds for s in got]
        assert starts == sorted(starts) and all(s.speaker_id == f"S{s.cluster + 1}" for s in got)
        if kw["exclusive_segments"]:
            assert all(a.end_time_seconds <= b.start_time_seconds for a, b in zip(got, got[1:]))
        assert all(s.end_time_seconds - s.start_time_seconds >= np.float32(kw["min_segment_duration"]) for s in got)
    # hand-checked cases: two chunks of 4 frames (0.5 s each), one local speaker each, both mapped to cluster 1
    w = np.zeros((2, 4, 2), np.float32)
    w[0, :, 0] = 0.9
    w[1, 2:, 1] = 0.8
    hard = np.array([[1, -2], [-2, 1]], np.int32)
    r = OfflineReconstruction(0.5, window_duration=2.0, min_segment_duration=0.0)
    segs = r.build_segments(w, hard, 2, [0.0, 2.0])
    assert [(s.cluster, s.start_time_seconds, s.end_time_seconds) for s in segs] == [(1, 0.0, 2.0), (1, 3.0, 4.0)]
    assert abs(segs[0].quality_score - 0.9) < 1e-6 and abs(segs[1].quality_score - 0.8) < 1e-6
    merged = OfflineReconstruction(0.5, window_duration=2.0, min_segment_duration=0.0, min_gap_duration=1.0) \
        .build_segments(w, hard, 2, [0.0, 2.0])
    assert [(s.cluster, s.start_time_seconds, s.end_time_seconds) for s in merged] == [(1, 0.0, 4.0)]
    assert abs(merged[0].quality_score - (0.9 * 2 + 0.8 * 1) / 3) < 1e-6          # duration-weighted blend
    assert OfflineReconstruction(0.0).build_segments(w, hard, 2) == []            # frameDuration <= 0 -> []
    assert OfflineReconstruction(0.5).build_segments(np.zeros((0, 0, 0), np.float32), [], 2) == []
    cents = np.random.default_rng(0).standard_normal((2, 7))
    db = OfflineReconstruction.build_speaker_database(merged + segs, cents)      # three segments, all of cluster 1
    odb, ocnt = oracle.build_speaker_database([s.cluster for s in merged + segs], cents)
    assert list(db) == ["S2"] and ocnt.tolist() == [0, 3] and db["S2"].tobytes() == odb[1].tobytes()
    c32 = cents[1].astype(np.float32)
    assert np.array_equal(db["S2"], ((c32 + c32) + c32) * np.float32(1.0 / 3.0))
    none = r.build_segments(w, np.full((2, 2), -2, np.int32), 2, [0.0, 2.0])
    assert all(s.cluster == 0 for s in none)     # zero votes everywhere: the ranking's tie-break picks cluster 0 (:177-186)
