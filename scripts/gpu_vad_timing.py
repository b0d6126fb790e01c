"""Times voice activity detection on the GPU: one 256 ms Silero tick (fa_vad_stream_model_inputs + advance, one
4096-sample chunk per session) at S = 1 / 64 / 512 / 4 096 sessions with host and device buffers, speech segmentation
of 10 000 five-minute clips (118 chunks each) and of one hour (879 chunks) with host and device buffers, and the FSMN-VAD decision over 64 one-hour
clips (360 000 frames each), beside the C++ oracle on one core.

    python scripts/gpu_vad_timing.py [--reps 50] [--out rows.jsonl]

Every call is timed on the host clock around the C call, which includes its synchronisation (every device-buffer
call ends in a device synchronise), p50 and p99 over `--reps` calls after two warm-up calls.  The model is left out: its
outputs are fixed arrays.  The oracle arm runs the same work one session or clip after another on one core inside
one native call (oracle_vad_tick, oracle_vad_segment_batch; one call per clip for FSMN), so it times the C++
restatement rather than Python, timed the same way.  The card's name and power limit are
read through NVML in the same process (queries only).  One JSON line per row on stdout, and in `--out` when given.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib                     # noqa: E402
from fluidaudio_b200 import vad as V                 # noqa: E402
from oracle import oracle_vad as O                   # noqa: E402


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
    except Exception as e:                           # the numbers still need their card
        return f"card not identified ({e})"


def timed(fn, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    a = np.asarray(ts) * 1e3
    return float(np.percentile(a, 50)), float(np.percentile(a, 99))


def clips_of(rng, n, P):
    levels = np.array([0.05, 0.25, 0.6, 0.8, 0.95], np.float32)
    return [np.repeat(rng.choice(levels, size=P), rng.integers(1, 12, size=P))[:P].astype(np.float32)
            for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out")
    a = ap.parse_args()
    _lib.set_device(0)
    where = card()
    rows = []

    def emit(**row):
        row["card"] = where
        rows.append(row)
        print(json.dumps(row), flush=True)

    rng = np.random.default_rng(0)
    L = _lib.load()
    cfg = V._c_config(None, None)
    ocfg = O.resolve(O.config())
    for S in (1, 64, 512, 4096):
        st = V.SileroVadStreams()
        ids = np.array([st.open() for _ in range(S)], np.int32)
        audio = rng.normal(0, 0.3, size=S * 4096).astype(np.float32)
        off = (np.arange(S + 1) * 4096).astype(np.int64)
        p = rng.uniform(size=S).astype(np.float32)
        nh, nc = rng.normal(size=(S, 128)).astype(np.float32), rng.normal(size=(S, 128)).astype(np.float32)
        inp, hid, cel = np.empty((S, 4160), np.float32), np.empty((S, 128), np.float32), np.empty((S, 128), np.float32)
        ev = np.empty((S, 2), np.int64)

        def host_tick():
            _lib.check(L.fa_vad_stream_model_inputs(st._h, S, ids.ctypes.data, audio.ctypes.data, off.ctypes.data,
                                                    inp.ctypes.data, hid.ctypes.data, cel.ctypes.data), "inputs")
            _lib.check(L.fa_vad_stream_advance(st._h, S, ids.ctypes.data, p.ctypes.data, nh.ctypes.data,
                                               nc.ctypes.data, C.byref(cfg), ev.ctypes.data), "advance")

        bufs = [_lib.DeviceBuffer(x.nbytes) for x in (audio, inp, hid, cel, p, nh, nc, ev)]
        for b, x in zip(bufs, (audio, inp, hid, cel, p, nh, nc, ev)):
            b.upload(x)
        d_audio, d_inp, d_hid, d_cel, d_p, d_nh, d_nc, d_ev = (b.ptr for b in bufs)

        def device_tick():
            _lib.check(L.fa_vad_stream_model_inputs_device(st._h, S, ids.ctypes.data, d_audio, off.ctypes.data, d_inp,
                                                           d_hid, d_cel), "inputs")
            _lib.check(L.fa_vad_stream_advance_device(st._h, S, ids.ctypes.data, d_p, d_nh, d_nc, C.byref(cfg),
                                                      d_ev), "advance")
            _lib.synchronize()

        for name, fn in (("host", host_tick), ("device", device_tick)):
            p50, p99 = timed(fn, a.reps)
            emit(workload="silero_tick", sessions=S, buffers=name, p50_ms=p50, p99_ms=p99)
        tick = O.Tick(S)
        p50, p99 = timed(lambda: tick.run(audio, off, p, nh, nc, ocfg), a.reps)
        emit(workload="silero_tick", sessions=S, buffers="oracle, one core, one native call", p50_ms=p50, p99_ms=p99)
        st.close_handle()

    for name, n, P in (("segment_10000x5min", 10000, 118), ("segment_1h", 1, 879)):
        reps = a.reps if n == 1 else max(5, a.reps // 5)
        flat = np.concatenate(clips_of(rng, n, P))
        off = (np.arange(n + 1) * P).astype(np.int64)
        totals = np.full(n, P * 4096, np.int64)
        counts, seg, total = np.zeros(n, np.int64), np.zeros((n * P, 2), np.int64), C.c_int64()
        d_in, d_seg = _lib.DeviceBuffer(flat.nbytes), _lib.DeviceBuffer(seg.nbytes)
        d_in.upload(flat)

        def host_segment():
            _lib.check(L.fa_vad_segment(flat.ctypes.data, off.ctypes.data, n, totals.ctypes.data, C.byref(cfg),
                                        counts.ctypes.data, seg.ctypes.data, n * P, C.byref(total)), "segment")

        def device_segment():
            _lib.check(L.fa_vad_segment_device(d_in.ptr, off.ctypes.data, n, totals.ctypes.data, C.byref(cfg),
                                               counts.ctypes.data, d_seg.ptr, n * P, C.byref(total)), "segment")
            _lib.synchronize()

        for buffers, fn in (("host", host_segment), ("device", device_segment)):
            p50, p99 = timed(fn, reps)
            emit(workload=name, clips=n, chunks=P, segments=total.value, buffers=buffers, p50_ms=p50, p99_ms=p99)
        p50, p99 = timed(lambda: O.segment_batch(flat, off, totals, ocfg), reps)
        emit(workload=name, clips=n, buffers="oracle, one core, one native call", p50_ms=p50, p99_ms=p99)

    runs = rng.integers(1, 3000, size=64 * 360_000 // 500 + 64)
    vals = rng.choice(np.array([0.05, 0.15, 0.25, 0.9], np.float32), size=runs.size)
    stream = np.repeat(vals, runs)
    sil = [stream[k * 360_000:(k + 1) * 360_000].astype(np.float32) for k in range(64)]
    p50, p99 = timed(lambda: V.fsmn_vad_decide(sil), max(5, a.reps // 5))
    emit(workload="fsmn_64x1h", clips=64, frames=360_000, segments=sum(map(len, V.fsmn_vad_decide(sil))),
         p50_ms=p50, p99_ms=p99)
    p50, p99 = timed(lambda: [O.fsmn_decide(x) for x in sil], 3)
    emit(workload="fsmn_64x1h", arm="oracle, one core, one native call per clip", p50_ms=p50, p99_ms=p99)
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
