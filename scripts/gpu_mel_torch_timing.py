"""Timing of the torch-style frontends (Cohere, StyleTTS2, LuxTTS) on the GPU, with the CPU oracle beside them.

Per frontend and workload (a 10 s prompt, a batch of 256 prompts of 3-12 s, one hour):
  device   CUDA-event time of fa_mel_compute_device (one clip) or fa_mel_compute_batch_device (the batch) on the preset
           handle, audio and rows resident in HBM (median of repeats);
  e2e      wall time of the class's host-buffer call (CohereMelSpectrogram.features, StyleTTS2MelExtractor.compute,
           LuxTtsMelExtractor.extract; the batch: fa_mel_compute_batch on the preset handle), median of repeats;
  oracle   wall time of oracle_mel_torch.cpp's single-threaded float32 restatement on this host (one run; the hour is
           extrapolated from 60 s and marked so).
Prints one JSON line per row.  Writes nothing.
"""
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from fluidaudio_b200 import _lib, synth   # noqa: E402
from fluidaudio_b200.mel import CohereMelSpectrogram, LuxTtsMelExtractor, StyleTTS2MelExtractor   # noqa: E402
from oracle import oracle_torch as O   # noqa: E402


def median_wall(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def device_ms(mel, audio, reps):
    n = audio.size
    d_a = _lib.DeviceBuffer(4 * n + 64)
    d_a.upload(audio)
    d_o = _lib.DeviceBuffer(4 * mel.n_mels * (n // mel.hop_length + 64))
    mel.compute_device(d_a, n, d_o)
    ts = []
    for _ in range(reps):
        mel.timer_start()
        mel.compute_device(d_a, n, d_o)
        ts.append(mel.timer_stop_ms())
    return float(np.median(ts))


def batch_device_ms(mel, clips, reps):
    offsets = np.zeros(len(clips) + 1, np.int64)
    offsets[1:] = np.cumsum([c.size for c in clips])
    packed = np.concatenate(clips)
    out_off = np.zeros(len(clips) + 1, np.int64)
    for i, c in enumerate(clips):
        out_off[i + 1] = out_off[i] + mel.frame_count(c.size) * mel.n_mels
    d_a, d_o = _lib.DeviceBuffer(4 * packed.size + 64), _lib.DeviceBuffer(4 * int(out_off[-1]) + 64)
    d_a.upload(packed)
    mel.compute_batch_device(d_a, offsets, d_o, out_off)
    ts = []
    for _ in range(reps):
        mel.timer_start()
        mel.compute_batch_device(d_a, offsets, d_o, out_off)
        ts.append(mel.timer_stop_ms())
    return float(np.median(ts))


def main():
    _lib.set_device(0)
    rng = np.random.default_rng(0)
    fronts = {
        "cohere": (CohereMelSpectrogram(), 16000, lambda e, a: e.features(a, 3500), O.cohere_compute),
        "styletts2": (StyleTTS2MelExtractor(), 24000, lambda e, a: e.compute(a), O.styletts2_compute),
        "luxtts": (LuxTtsMelExtractor(), 24000, lambda e, a: e.extract(a), O.luxtts_extract),
    }
    for name, (ext, rate, call, oracle_call) in fronts.items():
        mel = ext.mel
        prompt = synth.speech_like_audio(10 * rate, sample_rate=rate)
        clips = [synth.speech_like_audio(int(rng.integers(3 * rate, 12 * rate)), seed=i, sample_rate=rate)
                 for i in range(256)]
        hour = synth.tone_noise_audio(3600 * rate, sample_rate=rate)
        minute = hour[:60 * rate]
        rows = [
            ("10 s prompt", device_ms(mel, prompt, 20), median_wall(lambda: call(ext, prompt), 20),
             median_wall(lambda: oracle_call(prompt), 1), False),
            ("256 prompts", batch_device_ms(mel, clips, 10), median_wall(lambda: mel.compute_batch(clips), 5),
             median_wall(lambda: [oracle_call(c) for c in clips], 1), False),
            ("1 hour", device_ms(mel, hour, 5), median_wall(lambda: call(ext, hour), 3),
             60.0 * median_wall(lambda: oracle_call(minute), 1), True),
        ]
        for what, dev, e2e, cpu, extrapolated in rows:
            print(json.dumps({"frontend": name, "workload": what, "device_ms": round(dev, 4), "e2e_ms": round(e2e, 3),
                              "oracle_cpu_ms": round(cpu, 1), "oracle_extrapolated_from_60s": extrapolated}),
                  flush=True)


if __name__ == "__main__":
    main()
