"""End-to-end fa_audio_to_mel on one hour of 48 kHz stereo int16 and of 44.1 kHz mono float32 (the integer-rate sinc
paths: L = 1 and L = 160), for one or more builds of the library, run alternately in fresh processes, with the card's
name and power limit read in the same run.  Each build also prints a digest of its rows, so that builds which must
compute the same thing can be seen to.

    python scripts/gpu_resample_timing.py [--rounds 3] [--calls 10] [path/to/libfluidaudio_b200.so ...]

Without paths it times the tree's own build.
"""
import argparse
import hashlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(lib, calls):
    sys.path.insert(0, ROOT)
    import time
    import numpy as np
    from fluidaudio_b200 import _lib
    _lib.LIB_PATH = os.path.abspath(lib)
    from fluidaudio_b200.mel import AudioMelSpectrogram
    rng = np.random.default_rng(0)
    cases = (("48k stereo int16", 48000, rng.integers(-20000, 20000, (48000 * 3600, 2)).astype(np.int16), True),
             ("44.1k mono f32", 44100, rng.uniform(-0.6, 0.6, 44100 * 3600).astype(np.float32), False))
    m = AudioMelSpectrogram(n_mels=80)
    for what, rate, pcm, inter in cases:
        out = None
        for _ in range(2):      # warm-up: buffers, tables, module load
            out, _, _, _ = m.compute_from_pcm(pcm, rate, interleaved=inter)
        ts = []
        for _ in range(calls):  # the call ends in a device synchronise
            t0 = time.perf_counter()
            m.compute_from_pcm(pcm, rate, interleaved=inter, out=out)
            ts.append((time.perf_counter() - t0) * 1e3)
        digest = hashlib.sha256(out.tobytes()).hexdigest()[:16]
        # device time of the converter kernel alone, from a profiled run of its own (3 calls)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                m.compute_from_pcm(pcm, rate, interleaved=inter, out=out)
        us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
                 for e in prof.key_averages() if "sinc_kernel" in e.key) / 3
        print(f"{what:18s} median {np.median(ts):8.2f} ms  min {min(ts):8.2f} ms  sinc_kernel {us / 1e3:7.3f} ms"
              f"  rows {digest}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--child", default=None)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.calls)
        return
    libs = a.libs or [os.path.join(ROOT, "fluidaudio_b200", "lib", "libfluidaudio_b200.so")]
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip() or q.stderr.strip(), flush=True)
    for r in range(a.rounds):
        for lib in libs:
            print(f"-- round {r} {os.path.relpath(lib, ROOT)}", flush=True)
            subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lib, "--calls", str(a.calls)], check=True)


if __name__ == "__main__":
    main()
