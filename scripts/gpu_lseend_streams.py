"""Times one 100 ms tick of LS-EEND feature streams on the GPU: fa_lseend_stream_push (host buffers) and
fa_lseend_stream_push_device for S live sessions, against the same traffic as one fa_mel_lseend_features call per
session (the provider's popAllChunks slice of the tick, with the running mean carried on the host).

    python scripts/gpu_lseend_streams.py [--pushes 200] [--sessions 1,64,512,4096] [--out rows.jsonl]

Metadata: 16 kHz, 23 mels, hop 160, win 400 (nFFT 512), context 7, subsampling 10, chunk 1, conv delay 2, so one tick
of 1600 samples is one audio chunk and one model-input chunk per session.  A push is timed on the host clock around the
call and one device synchronisation (the device variant is asynchronous), p50 and p99 over `--pushes` ticks after 20
warm-up ticks.  The per-session row times the whole tick (S calls) over fewer ticks at large S.  The card's name and
power limit are read through NVML in the same process (queries only).  One JSON line per row on stdout, and in
`--out` when given.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib                                                          # noqa: E402
from fluidaudio_b200.lseend import LSEENDFeatureStreams, LSEENDStreamConfig               # noqa: E402
from fluidaudio_b200.mel import AudioMelSpectrogram, LogFloorMode                          # noqa: E402

TICK = 1600


def card():
    try:
        nvml = C.CDLL("libnvidia-ml.so.1")
        assert nvml.nvmlInit_v2() == 0
        h = C.c_void_p()
        assert nvml.nvmlDeviceGetHandleByIndex_v2(0, C.byref(h)) == 0
        name, mw = C.create_string_buffer(96), C.c_uint()
        nvml.nvmlDeviceGetName(h, name, 96)
        nvml.nvmlDeviceGetPowerManagementLimit(h, C.byref(mw))
        nvml.nvmlShutdown()
        return f"{name.value.decode()}, power limit {mw.value / 1000:.0f} W"
    except Exception as e:                                                                # the numbers still need their card
        return f"card not identified ({e})"


def pct(ts):
    a = np.sort(np.asarray(ts)) * 1e3
    return float(np.percentile(a, 50)), float(np.percentile(a, 99))


def run_streams(S, pushes, device, rng):
    cfg = LSEENDStreamConfig(sample_rate=16000, n_mels=23, hop_length=160, win_length=400, context_size=7,
                             subsampling=10, chunk_size=1, conv_delay=2)
    st = LSEENDFeatureStreams(cfg)
    ids = np.array([st.open() for _ in range(S)], np.int32)
    audio = (rng.standard_normal(S * TICK) * 0.1).astype(np.float32)
    offsets = np.arange(S + 1, dtype=np.int64) * TICK
    F, T = st.sizes.mel_frames * 23, cfg.chunk_size
    cap = 2 * S
    feats, masks, warm = np.empty(cap * F, np.float32), np.empty(cap * T, np.float32), np.empty(cap, np.int32)
    counts = np.zeros(S, np.int64)
    L, h = _lib.load(), st._h
    if device:
        d_audio = _lib.DeviceBuffer(audio.nbytes)
        d_audio.upload(audio)
        bufs = [_lib.DeviceBuffer(cap * F * 4), _lib.DeviceBuffer(cap * T * 4), _lib.DeviceBuffer(cap * 4)]

    def push():
        if device:
            _lib.check(L.fa_lseend_stream_push_device(h, S, ids.ctypes.data, d_audio.ptr, offsets.ctypes.data, None,
                                                      bufs[0].ptr, cap * F, bufs[1].ptr, cap * T, bufs[2].ptr, cap,
                                                      counts.ctypes.data), "push_device")
            _lib.synchronize()
        else:
            _lib.check(L.fa_lseend_stream_push(h, S, ids.ctypes.data, audio.ctypes.data, offsets.ctypes.data, None,
                                               feats.ctypes.data, feats.size, masks.ctypes.data, masks.size,
                                               warm.ctypes.data, warm.size, counts.ctypes.data), "push")

    for _ in range(20):
        push()
    ts, chunks = [], 0
    for _ in range(pushes):
        t0 = time.perf_counter()
        push()
        ts.append(time.perf_counter() - t0)
        chunks += int(counts.sum())
    st.close_handle()
    return ts, chunks


def run_per_session(S, ticks, rng):
    m = AudioMelSpectrogram(sample_rate=16000, n_mels=23, n_fft=512, hop_length=160, win_length=400, preemph=0.0,
                            pad_to=0, log_floor=1e-10, log_floor_mode=LogFloorMode.clamped, window_periodic=True)
    L = _lib.load()
    n = TICK + 512 - 160                                      # one audio chunk and its context
    slices = (rng.standard_normal((S, n)) * 0.1).astype(np.float32)
    means = np.zeros((S, 23), np.float32)
    cnt = [C.c_int64(0) for _ in range(S)]
    out = np.empty(10 * 23, np.float32)
    frames = C.c_int64()

    def tick():
        for i in range(S):
            _lib.check(L.fa_mel_lseend_features(m._h, slices[i].ctypes.data, n, means[i].ctypes.data, C.byref(cnt[i]),
                                                out.ctypes.data, out.size, C.byref(frames)), "fa_mel_lseend_features")

    for _ in range(3):
        tick()
    ts = []
    for _ in range(ticks):
        t0 = time.perf_counter()
        tick()
        ts.append(time.perf_counter() - t0)
    m.close()
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=200)
    ap.add_argument("--sessions", default="1,64,512,4096")
    ap.add_argument("--out", help="also write the rows to this file")
    a = ap.parse_args()
    assert _lib.device_count() >= 1, "needs an H100"
    _lib.set_device(0)
    gpu = card()
    rng = np.random.default_rng(0)
    with open(a.out or os.devnull, "w") as f:
        for S in (int(s) for s in a.sessions.split(",")):
            rows = []
            for device in (False, True):
                ts, chunks = run_streams(S, a.pushes, device, rng)
                p50, p99 = pct(ts)
                rows.append(dict(sessions=S, variant="push_device" if device else "push", p50_ms=p50, p99_ms=p99,
                                 chunks_per_push=chunks / a.pushes))
            ticks = max(5, min(100, 2000 // S))
            p50, p99 = pct(run_per_session(S, ticks, rng))
            rows.append(dict(sessions=S, variant="fa_mel_lseend_features per session", p50_ms=p50, p99_ms=p99,
                             ticks=ticks))
            for r in rows:
                r["card"] = gpu
                line = json.dumps(r)
                print(line, flush=True)
                f.write(line + "\n")


if __name__ == "__main__":
    main()
