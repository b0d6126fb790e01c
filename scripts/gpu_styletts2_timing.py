"""StyleTTS2 synthesis glue timing on the GPU: p50 / p99 per call, each with its synchronisation, of
fa_styletts2_sampler_inputs, fa_styletts2_style and fa_styletts2_align at R = 1 / 64 / 512 / 1 024 requests of about
100 tokens (bucket 128) with C = 50 duration logits, dC = 640 and tC = 512, about 6 frames per token, with host and
device buffers; align's bytes (its reads and its en / asr writes) over its device-buffer p50 beside the H100's
3.35 TB/s; and the C++ oracle doing one request's glue on one core.  The card name and power limit are read in the
same run.

    python scripts/gpu_styletts2_timing.py [--reps 10] [--sizes 1,64,512,1024]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fluidaudio_b200 import _lib  # noqa: E402
from fluidaudio_b200 import styletts2 as S  # noqa: E402
from oracle import oracle_styletts2 as O  # noqa: E402

C_, DC, TC, BUCKET = 50, 640, 512, 128


def pct(ts):
    ts = np.sort(np.array(ts) * 1e3)
    return ts[len(ts) // 2], ts[min(len(ts) - 1, int(0.99 * len(ts)))]


def inputs(R):
    rng = np.random.default_rng(R)
    counts = rng.integers(95, 106, size=R).astype(np.int32)
    W = int(counts.max())
    ids = rng.integers(1, 178, size=int(counts.sum())).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    dur = rng.integers(3, 10, size=(R, W))
    logits = (np.where(np.arange(C_)[None, None, :] < dur[:, :, None], 30.0, -30.0) +
              rng.normal(size=(R, W, C_))).astype(np.float32)
    d = rng.normal(size=(R, W, DC)).astype(np.float32)
    t = rng.normal(size=(R, TC, W)).astype(np.float32)
    p, r = rng.normal(size=(R, 256)).astype(np.float32), rng.normal(size=(R, 256)).astype(np.float32)
    return counts, W, ids, off, logits, d, t, p, r


def run(R, reps, device, frame_stride=None):
    L = _lib.load()
    glue = S.StyleTTS2Glue()
    counts, W, ids, off, logits, d, t, p, r = inputs(R)
    seeds = np.arange(R, dtype=np.uint64)
    ab = np.full(R, 0.3, np.float32), np.full(R, 0.7, np.float32)
    if frame_stride is None:
        frame_stride = int(glue.align([logits[i, :counts[i]] for i in range(R)], [d[i, :counts[i]] for i in range(R)],
                                      [t[i, :, :counts[i]] for i in range(R)])[2].max())
    host = {"tokens": np.empty((R, BUCKET), np.int32), "mask": np.empty((R, BUCKET), np.int32),
            "noise": np.empty((R, 5, 256), np.float32), "ref": np.empty((R, 128), np.float32),
            "s": np.empty((R, 128), np.float32), "en": np.empty((R, DC, frame_stride), np.float32),
            "asr": np.empty((R, TC, frame_stride), np.float32)}
    ins = {"ids": ids, "logits": logits, "d": d, "t": t, "p": p, "r": r}
    if device:
        bufs = {k: _lib.DeviceBuffer(a.nbytes) for k, a in list(host.items()) + list(ins.items())}
        for k, a in ins.items():
            bufs[k].upload(a)
        P = {k: b.ptr for k, b in bufs.items()}
    else:
        P = {k: a.ctypes.data for k, a in list(host.items()) + list(ins.items())}
    sfx = "_device" if device else ""
    reasons, frames = np.zeros(R, np.int32), np.zeros(R, np.int64)
    durs = np.zeros(int(counts.sum()), np.int32)
    times = {k: [] for k in ("sampler inputs", "style", "align")}
    _lib.synchronize()
    for rep in range(reps + 1):
        def timed(key, fn):
            t0 = time.perf_counter()
            _lib.check(fn(), key)
            _lib.synchronize()
            if rep:
                times[key].append(time.perf_counter() - t0)
        timed("sampler inputs", lambda: getattr(L, "fa_styletts2_sampler_inputs" + sfx)(
            R, P["ids"], off.ctypes.data, seeds.ctypes.data, BUCKET, P["tokens"], P["mask"], P["noise"],
            reasons.ctypes.data))
        timed("style", lambda: getattr(L, "fa_styletts2_style" + sfx)(
            R, P["p"], P["r"], ab[0].ctypes.data, ab[1].ctypes.data, P["ref"], P["s"]))
        timed("align", lambda: getattr(L, "fa_styletts2_align" + sfx)(
            R, counts.ctypes.data, P["logits"], C_, C_, W * C_, P["d"], DC, DC, W * DC, P["t"], TC, W, TC * W,
            frame_stride, P["en"], P["asr"], frames.ctypes.data, durs.ctypes.data, reasons.ctypes.data))
    if device:
        for b in bufs.values():
            b.free()
    read = int(counts.sum()) * (C_ + DC + TC) * 4
    written = R * (DC + TC) * frame_stride * 4
    return times, read + written, frame_stride, float(frames.mean())


def oracle_time(reps=5):
    """one request's glue on one core: sampler inputs, blend, durations, alignment, both matmuls, transpose, shifts"""
    counts, W, ids, off, logits, d, t, p, r = inputs(1)
    n = int(counts[0])
    t0 = time.perf_counter()
    for _ in range(reps):
        O.sampler_inputs(ids[:n], BUCKET, 1)
        O.blend(p[0], r[0], 0.3, 0.7)
        O.align(logits[0, :n], d[0, :n], t[0, :, :n])
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="1,64,512,1024")
    a = ap.parse_args()
    _lib.set_device(0)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    for R in (int(s) for s in a.sizes.split(",")):
        for device in (False, True):
            t, nbytes, stride, mean_f = run(R, a.reps, device)
            cells = "  ".join(f"{k} {pct(v)[0]:.3f}/{pct(v)[1]:.3f}" for k, v in t.items())
            rate = nbytes / (pct(t["align"])[0] * 1e-3) / 1e12
            print(f"R={R:5d} {'device' if device else 'host  '}  p50/p99 ms: {cells}  | align {nbytes / 1e6:.1f} MB "
                  f"(frame_stride {stride}, mean F {mean_f:.0f}) = {rate:.2f} TB/s of 3.35")
    print(f"oracle one core, one request's glue: {oracle_time() * 1e3:.1f} ms")


if __name__ == "__main__":
    main()
