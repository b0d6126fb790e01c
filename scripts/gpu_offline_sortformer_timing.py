"""Offline Sortformer windows timing on the GPU: fa_offline_sortformer_model_inputs_device and
fa_offline_sortformer_stitch_device with device buffers for 1 000 clips of 30 s (one window each) and 64 files of one
hour (159 windows each), each timed over repeated calls after a warm-up between device synchronisations; model_inputs' bytes (the
mel rows it reads, the windows and lengths it writes) over its time beside the H100's 3.35 TB/s; the stitch time per
file of the hour case; and the C++ oracle's window loop for one hour on one core.  The card name and power limit are
read in the same run.

    python scripts/gpu_offline_sortformer_timing.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fluidaudio_b200 import _lib  # noqa: E402
from fluidaudio_b200.offline_sortformer import OfflineSortformerWindows  # noqa: E402
from oracle import oracle_offline_sortformer as O  # noqa: E402

HBM = 3.35e12


def call_ms(fn, reps):
    """mean time per call over `reps` calls after a warm-up, on the host clock between device synchronisations (the
    calls run on the library's own stream, which events recorded on torch's stream would not bracket)"""
    fn()
    _lib.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    _lib.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def case(name, frames, reps):
    win = OfflineSortformerWindows()
    frames = np.asarray(frames, np.int64)
    w, r = win.plan(frames, 100)
    W, R = int(w.sum()), int(r.sum())
    offsets = np.concatenate([[0], np.cumsum(frames * 128)])[:-1].astype(np.int64)
    mel = torch.randn(int(frames.sum()) * 128, device="cuda")
    out = torch.empty(W * 128 * 3072, device="cuda")
    lens = torch.empty(W, dtype=torch.int32, device="cuda")
    preds = torch.rand(W * 384 * 4, device="cuda")
    rows = torch.empty(R * 4, device="cuda")
    torch.cuda.synchronize()
    mi = call_ms(lambda: win.model_inputs_device(mel.data_ptr(), offsets, frames, W, out.data_ptr(),
                                                   lens.data_ptr(), 100), reps)
    st = call_ms(lambda: win.stitch_device(preds.data_ptr(), frames, rows.data_ptr(), None, 100), reps)
    moved = int(frames.sum()) * 128 * 4 + W * 128 * 3072 * 4 + W * 4
    print(f"{name}: {len(frames)} files, {W} windows, {R} rows | model_inputs {mi:.3f} ms, "
          f"{moved / 1e9:.2f} GB moved, {moved / mi / 1e9:.3f} TB/s = {moved / mi / 1e-3 / HBM * 100:.1f}% of 3.35 TB/s"
          f" | stitch {st:.3f} ms ({st * 1e3 / len(frames):.1f} us per file of the call)", flush=True)
    return mi, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    _lib.set_device(0)
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip(), flush=True)
    case("30 s clips", [3001] * 1000, a.reps)
    case("one-hour files", [360_001] * 64, a.reps)
    case("one one-hour file", [360_001], a.reps)
    rows = np.random.default_rng(0).normal(size=(360_001, 128)).astype(np.float32)
    zeros = np.zeros((384, 4), np.float32)
    t0 = time.perf_counter()
    O.stitch(rows, 360_001, 100, lambda mel, ml: zeros)
    print(f"oracle window loop (copy + stitch, model returning zeros), one hour on one core: "
          f"{(time.perf_counter() - t0) * 1e3:.1f} ms", flush=True)


if __name__ == "__main__":
    main()
