"""Live log-mel streams on one H100: fa_mel_stream_push against a loop of per-session fa_mel_compute calls.

Traffic: S sessions (1, 64, 512, 4096) each receiving one chunk per push (1 600 samples = a 100 ms mic callback, and
10 080 samples), 128 mels, both transform precisions, host buffers in and out.  Per push (host clock around a call that
ends in a synchronise): p50 / p99 over at least --seconds, frames/s and kernel launches per push.  Real-time capacity: the
largest S whose p99 push time stays under the chunk's audio duration.  The same traffic as the reference's host sequence
(per session: buffer, .prePadded fa_mel_compute with expected_frames, drop consumed samples) is timed per tick over all
sessions and its rows compared with the stream's for equality.  Prints one JSON line per case; --out FILE also writes
them to FILE as one JSON list.

    python scripts/gpu_mel_stream.py [--seconds 1.0] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fluidaudio_b200 import _lib, synth   # noqa: E402
from fluidaudio_b200.mel import AudioMelSpectrogram, MelStreams, Precision   # noqa: E402

RATE = 16000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


class Traffic:
    """Pre-packed pushes: push t gives session i samples [t*chunk, (t+1)*chunk) of its own signal."""

    def __init__(self, S, chunk, pushes):
        self.S, self.chunk = S, chunk
        base = synth.tone_noise_audio(chunk * (pushes + S), seed=1)
        self.audio = [np.ascontiguousarray(np.concatenate([base[(t + i) * chunk:(t + i + 1) * chunk] for i in range(S)]))
                      for t in range(pushes)]
        self.offsets = np.arange(S + 1, dtype=np.int64) * chunk


def stream_push(L, m, ids, audio, offsets, out, frames):
    st = L.fa_mel_stream_push(m._h, ids.size, ids.ctypes.data, audio.ctypes.data, offsets.ctypes.data, None,
                              out.ctypes.data, out.size, frames.ctypes.data)
    if st != 0:
        raise _lib.FluidAudioError(st, "fa_mel_stream_push", L.fa_last_error().decode())


def loop_tick(L, m, sessions, audio, chunk, out):
    """The reference's host sequence for every session of one tick; returns the rows (concatenated in session order)."""
    M, hop, hw = m.n_mels, m.hop_length, m.win_length // 2
    rows = 0
    ml, nf = C.c_int64(), C.c_int64()
    for i, s in enumerate(sessions):
        s["buf"] = np.concatenate([s["buf"], audio[i * chunk:(i + 1) * chunk]])
        s["received"] += chunk
        count = (s["received"] - hw) // hop + 1 - s["emitted"] if s["received"] >= hw else 0
        if count <= 0:
            continue
        st = L.fa_mel_compute(m._h, s["buf"].ctypes.data, s["buf"].size, float(s["last"]), 1, count, 0,
                              out[rows * M:].ctypes.data, (out.size // M - rows) * M, C.byref(ml), C.byref(nf))
        assert st == 0 and ml.value == count
        rows += count
        s["last"] = s["buf"][count * hop - 1]
        s["buf"] = s["buf"][count * hop:]
        s["emitted"] += count
    return out[:rows * M]


def run_case(L, prec, S, chunk, seconds, loop_ticks):
    m = AudioMelSpectrogram(n_mels=128, precision=prec)
    streams = MelStreams(m)
    ids = np.array([streams.open() for _ in range(S)], np.int32)
    pushes = int(max(4, min(64, 200_000_000 // (S * chunk))))   # pre-packed pushes, cycled
    tr = Traffic(S, chunk, pushes)
    out = np.empty((chunk // m.hop_length + 2) * S * m.n_mels, np.float32)
    frames = np.zeros(S, np.int64)
    for t in range(3):   # warm-up (allocations, modules)
        stream_push(L, m, ids, tr.audio[t], tr.offsets, out, frames)
    times, rows, launches, t = [], 0, 0, 3
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(times) < 20:
        a = tr.audio[t % pushes]
        l0 = _lib.kernel_launch_count()
        t0 = time.perf_counter()
        stream_push(L, m, ids, a, tr.offsets, out, frames)
        times.append(time.perf_counter() - t0)
        launches = max(launches, _lib.kernel_launch_count() - l0)
        rows += int(frames.sum())
        t += 1
    times = np.array(times)
    res = dict(precision=prec.name, sessions=S, chunk=chunk, pushes=len(times),
               push_p50_us=round(float(np.percentile(times, 50)) * 1e6, 1),
               push_p99_us=round(float(np.percentile(times, 99)) * 1e6, 1),
               frames_per_s=round(rows / float(times.sum())), max_launches_per_push=int(launches),
               realtime=bool(np.percentile(times, 99) < chunk / RATE))
    # the same traffic as per-session calls, fresh sessions on both sides, rows compared for equality
    streams2 = MelStreams(AudioMelSpectrogram(n_mels=128, precision=prec))
    ids2 = np.array([streams2.open() for _ in range(S)], np.int32)
    sess = [dict(buf=np.zeros(m.n_fft // 2, np.float32), last=np.float32(0), received=0, emitted=0) for _ in range(S)]
    lout = np.empty_like(out)
    equal, tick_times = True, []
    for k in range(loop_ticks):
        t0 = time.perf_counter()
        ref = loop_tick(L, m, sess, tr.audio[k], chunk, lout)
        tick_times.append(time.perf_counter() - t0)
        stream_push(L, streams2.mel, ids2, tr.audio[k], tr.offsets, out, frames)
        got = out[:int(frames.sum()) * m.n_mels]
        equal = equal and got.shape == ref.shape and np.array_equal(got, ref)
    res.update(loop_tick_p50_us=round(float(np.median(tick_times)) * 1e6, 1), loop_ticks=loop_ticks,
               loop_equal=bool(equal))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--sessions", default="1,64,512,4096")
    ap.add_argument("--chunks", default="1600,10080")
    ap.add_argument("--out", default=None, help="also write every result to this JSON file")
    args = ap.parse_args()
    assert _lib.device_count() >= 1, "needs an sm_90a GPU"
    L = _lib.load()
    gpu = card()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    results = []
    for prec in (Precision.f32, Precision.f64):
        for chunk in (int(c) for c in args.chunks.split(",")):
            cap = 0
            for S in (int(s) for s in args.sessions.split(",")):
                r = run_case(L, prec, S, chunk, args.seconds, loop_ticks=8 if S <= 512 else 3)
                r["gpu"] = gpu
                print(json.dumps(r), flush=True)
                results.append(r)
                if r["realtime"]:
                    cap = S
            summary = dict(precision=prec.name, chunk=chunk, realtime_capacity_sessions=cap, gpu=gpu)
            print(json.dumps(summary), flush=True)
            results.append(summary)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
