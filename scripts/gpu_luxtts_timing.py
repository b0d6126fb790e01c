"""LuxTTS synthesis timing on the GPU: p50 / p99 per call, each with its synchronisation, at R = 1 / 64 / 512 / 1 024
requests of 5 s prompts whose generated span fills the 555-frame vocoder bucket (the longest output a request can
have: 554 x 512 samples, 5.9 s at 48 kHz), with host and device buffers, beside the C++ oracle doing the same work on
one core.  The card name and power limit are read in the same run.

    python scripts/gpu_luxtts_timing.py [--reps 10] [--sizes 1,64,512,1024]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fluidaudio_b200 import _lib  # noqa: E402
from fluidaudio_b200 import luxtts as LX  # noqa: E402
from oracle import oracle_luxtts as O  # noqa: E402

PT, TT = 60, 71   # 469 prompt frames / 60 tokens * 71 tokens = 555 generated frames


def pct(ts):
    ts = np.sort(np.array(ts) * 1e3)
    return ts[len(ts) // 2], ts[min(len(ts) - 1, int(0.99 * len(ts)))]


def run(R, reps, device):
    L = _lib.load()
    rng = np.random.default_rng(R)
    prompts = [(rng.normal(size=120000) * 0.05).astype(np.float32) for _ in range(R)]
    audio = np.concatenate(prompts)
    off = np.arange(R + 1, dtype=np.int64) * 120000
    pt, tt = np.full(R, PT, np.int32), np.full(R, TT, np.int32)
    sp, sd = np.ones(R, np.float32), np.arange(R, dtype=np.uint64)
    emb = rng.normal(size=(R, 256, 100)).astype(np.float32)
    v = rng.normal(size=(R, 1024, 100)).astype(np.float32)
    voc = rng.normal(size=(R, 554 * 512)).astype(np.float32)
    h = LX.LuxTtsRequests()
    reasons, ids = np.zeros(R, np.int32), np.zeros(R, np.int32)
    plans = (_lib.LuxTtsPlanInfo * R)()
    host = {k: np.empty(n, np.float32) for k, n in (("sc", R * 102400), ("pm", R * 1024), ("tc", R * 102400),
                                                    ("x", R * 102400), ("t", R), ("mel", R * 100 * 555),
                                                    ("out", R * 554 * 512))}
    if device:
        bufs = {k: _lib.DeviceBuffer(a.nbytes) for k, a in host.items()}
        d_in = {k: _lib.DeviceBuffer(a.nbytes) for k, a in (("audio", audio), ("emb", emb), ("v", v), ("voc", voc))}
        for k, a in (("audio", audio), ("emb", emb), ("v", v), ("voc", voc)):
            d_in[k].upload(a)
        P = {k: b.ptr for k, b in bufs.items()}
        I = {k: b.ptr for k, b in d_in.items()}
    else:
        P = {k: a.ctypes.data for k, a in host.items()}
        I = {"audio": audio.ctypes.data, "emb": emb.ctypes.data, "v": v.ctypes.data, "voc": voc.ctypes.data}
    sfx = "_device" if device else ""
    times = {k: [] for k in ("begin", "text condition", "step", "vocoder input", "finish")}
    lengths, total = np.zeros(R, np.int64), C.c_int64()
    _lib.synchronize()
    for rep in range(reps + 1):
        def timed(key, fn):
            t0 = time.perf_counter()
            _lib.check(fn(), key)
            _lib.synchronize()
            if rep:
                times[key].append(time.perf_counter() - t0)
        timed("begin", lambda: getattr(L, "fa_luxtts_begin" + sfx)(
            h._h, R, I["audio"], off.ctypes.data, pt.ctypes.data, tt.ctypes.data, sp.ctypes.data, sd.ctypes.data,
            reasons.ctypes.data, ids.ctypes.data, plans, P["sc"], P["pm"]))
        timed("text condition", lambda: getattr(L, "fa_luxtts_text_condition" + sfx)(
            h._h, R, ids.ctypes.data, I["emb"], 100, 25600, P["tc"]))
        for _ in range(4):
            def step():
                st = getattr(L, "fa_luxtts_model_inputs" + sfx)(h._h, R, ids.ctypes.data, P["x"], P["t"])
                return st or getattr(L, "fa_luxtts_advance" + sfx)(h._h, R, ids.ctypes.data, I["v"], 100, 102400)
            timed("step", step)
        timed("vocoder input", lambda: getattr(L, "fa_luxtts_vocoder_input" + sfx)(h._h, R, ids.ctypes.data, 555,
                                                                                  P["mel"]))
        timed("finish", lambda: getattr(L, "fa_luxtts_finish" + sfx)(
            h._h, R, ids.ctypes.data, I["voc"], 554 * 512, 554 * 512, P["out"], R * 554 * 512, lengths.ctypes.data,
            C.byref(total)))
    assert all(p.bucket == 555 and p.gen_frames == 555 for p in plans)
    h.close_handle()
    return times


def oracle_time(R):
    """the oracle's work for R requests on one core: RMS, gain, noise, four steps, vocoder input and finish (the prompt
    mel is not part of it)"""
    rng = np.random.default_rng(R)
    p = (rng.normal(size=120000) * 0.05).astype(np.float32)
    v = rng.normal(size=102400).astype(np.float32)
    voc = rng.normal(size=554 * 512).astype(np.float32)
    reps = max(1, min(R, 8))
    t0 = time.perf_counter()
    for i in range(reps):
        r = O.rms(p)
        O.gain(p, r)
        x = O.noise(i, 1024 * 100)
        for k in range(4):
            x = O.step(x, v, k)
        O.vocoder_input(x, 469, 555, 555)
        O.finish(voc, 555, r)
    return (time.perf_counter() - t0) / reps * R


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
            t = run(R, a.reps, device)
            cells = "  ".join(f"{k} {pct(v)[0]:.3f}/{pct(v)[1]:.3f}" for k, v in t.items())
            print(f"R={R:5d} {'device' if device else 'host  '}  p50/p99 ms: {cells}")
        print(f"R={R:5d} oracle one core: {oracle_time(R) * 1e3:.1f} ms per pass (begin..finish, no mel)")


if __name__ == "__main__":
    main()
