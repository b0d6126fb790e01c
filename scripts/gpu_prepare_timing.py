"""Times fa_seg_decode_device and fa_embedding_plan_device at the size of one hour of audio (community preset: 10 s windows,
589 frames, 7 classes; step ratios 0.2 and 0.1) and prints each call's time beside the bytes its algorithm moves.

    python scripts/gpu_prepare_timing.py            (needs the H100; there is no fallback)

Each call is timed as the library's device timer sees it (CUDA events around `reps` calls after warm-up, `reps` chosen so
that the window is at least a second).  A call includes its launches, the upload of the per-chunk descriptors, the
read-back of its counters and one stream synchronisation, so the figure is the call's time, not a kernel's: the rate printed
beside the 3.35 TB/s of the H100 SXM data sheet is algorithmic bytes (from shapes) over call time.  The card's name and
power limit are read through NVML in the same process (queries only).
"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib, synth                                             # noqa: E402
from fluidaudio_b200.segmentation import (EmbeddingPlanConfig, OfflineEmbeddingPlanner, OfflineSegmentationProcessor,  # noqa: E402
                                          SegmentationConfig)

DATA_SHEET_TBS = 3.35


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
    except Exception as e:                                                          # the numbers still need their card
        return f"card not identified ({e})"


def timed(fn, min_seconds=1.0):
    L = _lib.load()
    for _ in range(5):
        fn()
    reps, ms = 10, C.c_float()
    while True:
        _lib.check(L.fa_timer_start(), "fa_timer_start")
        for _ in range(reps):
            fn()
        _lib.check(L.fa_timer_stop_ms(C.byref(ms)), "fa_timer_stop_ms")
        if ms.value >= 1000.0 * min_seconds:
            return ms.value / reps, reps
        reps = int(reps * max(2.0, 1100.0 * min_seconds / max(ms.value, 1e-3)))


def main():
    assert _lib.device_count() >= 1, "needs an H100"
    _lib.set_device(0)
    print("card:", card())
    frames, classes = 589, 7
    for ratio in (0.2, 0.1):
        seg_cfg = SegmentationConfig(step_ratio=ratio)
        logits, truth = synth.segmentation_logits(3600.0, speakers=3, seed=1, step_ratio=ratio)
        chunks = logits.shape[0]
        proc, planner = OfflineSegmentationProcessor(seg_cfg), OfflineEmbeddingPlanner(seg_cfg, EmbeddingPlanConfig())
        d_logits, d_lp = _lib.DeviceBuffer(logits.nbytes), _lib.DeviceBuffer(logits.nbytes)
        d_w = _lib.DeviceBuffer(chunks * frames * 3 * 4)
        d_logits.upload(logits)
        ms, reps = timed(lambda: proc.decode_device(d_logits, chunks, frames, classes, d_lp, d_w))
        moved = logits.nbytes * 2 + chunks * frames * 3 * 4
        print(f"step ratio {ratio}: {chunks} chunks | fa_seg_decode_device {ms * 1e3:8.1f} us per call over {reps} calls, "
              f"{moved / 1e6:.1f} MB in + out -> {moved / ms / 1e9:.3f} TB/s (data sheet {DATA_SHEET_TBS} TB/s)")
        cap = chunks * 3
        sizes = dict(chunk_index=4, speaker_index=4, start_frame=4, end_frame=4, start_time=8, end_time=8, mask_sum=4,
                     used_fallback=4, reuse_of=4, frame_weights=4 * frames, model_weights=4 * planner.config.weight_frames)
        d_out = {k: _lib.DeviceBuffer(cap * v) for k, v in sizes.items()}
        args = (d_w, chunks, frames, 3, truth["chunk_offsets"], 10.0 / frames, truth["total_samples"], d_out)
        entries, counters = planner.plan_device(*args)
        ms, reps = timed(lambda: planner.plan_device(*args))
        moved = 2 * chunks * frames * 3 * 4 + entries * sum(sizes.values())     # weights read by both kernels, rows written
        print(f"step ratio {ratio}: {entries} entries {counters} | fa_embedding_plan_device {ms * 1e3:8.1f} us per call over "
              f"{reps} calls, {moved / 1e6:.1f} MB -> {moved / ms / 1e9:.3f} TB/s (data sheet {DATA_SHEET_TBS} TB/s)")


if __name__ == "__main__":
    main()
