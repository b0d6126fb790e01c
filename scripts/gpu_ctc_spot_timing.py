"""Times CTC keyword spotting on the GPU: the spotter over one hour of log-probs (45 000 frames x 1025, 80 ms frames)
with K = 100 and K = 1 000 terms of 1-8 tokens beside the C++ oracle's one-term-after-another loop on one core, 64
clips x 5 min with K = 256, 10 000 constrained queries of 2 s windows, and fa_ctc_log_softmax over the hour.

    python scripts/gpu_ctc_spot_timing.py [--reps 10] [--oracle-terms 10] [--out rows.jsonl]

Every call is timed on the host clock around the call and a device synchronisation, with the inputs and outputs in
HBM (the _device variants), p50 and p99 over `--reps` calls after two warm-up calls.  The oracle arm times the first
`--oracle-terms` terms one after another on one core, as the reference loops over its vocabulary, and scales that to
the whole vocabulary; its row says so.  The card's name and power limit are read through NVML in the same process
(queries only).  One JSON line per row on stdout, and in `--out` when given.
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
from fluidaudio_b200 import ctc_spotting as S        # noqa: E402
from oracle import oracle_ctc as O                   # noqa: E402

V, BLANK = 1025, 1024


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
        _lib.synchronize()
        ts.append(time.perf_counter() - t0)
    a = np.asarray(ts) * 1e3
    return float(np.percentile(a, 50)), float(np.percentile(a, 99))


def log_probs(rng, T):
    return S.apply_log_softmax(rng.normal(0, 3, size=(T, V)).astype(np.float32), BLANK)


def terms(rng, K):
    return [[int(x) for x in rng.integers(0, BLANK, size=int(rng.integers(1, 9)))] for _ in range(K)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--oracle-terms", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert _lib.device_count() >= 1, "needs an H100"
    _lib.set_device(0)
    rng = np.random.default_rng(0)
    where = card()
    rows = []

    def emit(**row):
        row["card"] = where
        rows.append(row)
        print(json.dumps(row), flush=True)

    hour = log_probs(rng, 45000)
    d_hour = _lib.DeviceBuffer(hour.nbytes)
    d_hour.upload(hour)
    off = np.array([0, 45000], np.int64)
    for K in (100, 1000):
        vocab = terms(rng, K)
        sp = S.CtcSpotter(V, vocab, BLANK)
        cap = 45000 * K // 2 + 2 * K
        d_det = _lib.DeviceBuffer(cap * _lib.CTC_DETECTION.itemsize)
        st, _, total = sp.spot_device(d_hour, off, d_det, cap)
        p50, p99 = timed(lambda: sp.spot_device(d_hour, off, d_det, cap), a.reps)
        sub = vocab[:a.oracle_terms]
        t0 = time.perf_counter()
        for tok in sub:
            O.word_spot_multiple(hour, tok, O.threshold(None, len(tok)), BLANK)
        cpu = (time.perf_counter() - t0) * 1e3 * K / len(sub)
        emit(workload=f"spot 45000x1025, K={K}", detections=total, gpu_p50_ms=p50, gpu_p99_ms=p99,
             oracle_one_core_ms=cpu, oracle_note=f"timed over the first {len(sub)} terms, scaled to {K}")
        sp.close()
    # 64 clips x 5 min (3 750 frames each) with K = 256
    clips = np.concatenate([log_probs(rng, 3750) for _ in range(64)])
    d_clips = _lib.DeviceBuffer(clips.nbytes)
    d_clips.upload(clips)
    off64 = np.arange(65, dtype=np.int64) * 3750
    sp = S.CtcSpotter(V, terms(rng, 256), BLANK)
    cap = 64 * 256 * 1877
    d_det = _lib.DeviceBuffer(cap * _lib.CTC_DETECTION.itemsize)
    st, _, total = sp.spot_device(d_clips, off64, d_det, cap)
    p50, p99 = timed(lambda: sp.spot_device(d_clips, off64, d_det, cap), a.reps)
    emit(workload="spot 64 clips x 3750x1025, K=256", detections=total, gpu_p50_ms=p50, gpu_p99_ms=p99)
    sp.close()
    # 10 000 constrained queries of 2 s (25-frame) windows over the hour
    Q = 10000
    queries = terms(rng, Q)
    tok = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in queries]), np.int32)
    toff = np.concatenate([[0], np.cumsum([len(t) for t in queries])]).astype(np.int64)
    ss = np.ascontiguousarray(rng.integers(0, 45000 - 25, size=Q), np.int64)
    se = np.ascontiguousarray(ss + 25, np.int64)
    d_s, d_a, d_e = _lib.DeviceBuffer(4 * Q), _lib.DeviceBuffer(8 * Q), _lib.DeviceBuffer(8 * Q)
    L = _lib.load()

    def constrained():
        _lib.check(L.fa_ctc_spot_constrained_device(d_hour.ptr, 45000, V, BLANK, Q, _lib.ptr(tok), _lib.ptr(toff),
                                                    _lib.ptr(ss), _lib.ptr(se), d_s.ptr, d_a.ptr, d_e.ptr), "constrained")
    p50, p99 = timed(constrained, a.reps)
    emit(workload="constrained 10000 queries x 25 frames", gpu_p50_ms=p50, gpu_p99_ms=p99)
    # fa_ctc_log_softmax_device over the hour
    logits = rng.normal(0, 3, size=(45000, V)).astype(np.float32)
    d_logits, d_out = _lib.DeviceBuffer(logits.nbytes), _lib.DeviceBuffer(logits.nbytes)
    d_logits.upload(logits)

    def softmax():
        _lib.check(L.fa_ctc_log_softmax_device(d_logits.ptr, 45000, V, 0, 1.0, 0.0, BLANK, d_out.ptr), "softmax")
    p50, p99 = timed(softmax, a.reps)
    emit(workload="log_softmax 45000x1025", gpu_p50_ms=p50, gpu_p99_ms=p99)
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
