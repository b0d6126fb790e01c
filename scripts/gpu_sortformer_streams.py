"""Times one Sortformer chunk tick on the GPU: fa_sortformer_update (+ fa_sortformer_model_inputs) for S live sessions,
device and host-buffer variants, against the CPU oracle's single-threaded streamingUpdate per session.

    python scripts/gpu_sortformer_streams.py [--pushes 40] [--sessions 1,64,512,4096] [--presets default,balancedV2]

Sessions are warmed through their first compressions and staggered, so that every tick has sessions popping and
compressing as a live deployment does.  A push is timed on the host clock around the call and one device
synchronisation (the device variant is asynchronous), p50 and p99 over `--pushes` pushes after warm-up; the model-input
gather is timed the same way and added.  The oracle row is the restatement's per-session update time (C++, -O2, one
thread, called through ctypes) on 64 sessions in the same steady state, times S.  The card's name and power limit are
read through NVML in the same process (queries only).  One JSON line per row.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib                                                   # noqa: E402
from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams         # noqa: E402

D, S4 = 512, 4


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


def inputs(cfg, n, rng):
    rows = cfg.chunk_left_context + cfg.chunk_len + cfg.chunk_right_context
    pred_rows = cfg.spkcache_len + cfg.fifo_len + rows
    E = rng.normal(size=(n, rows, D)).astype(np.float32)
    P = rng.uniform(0.0, 1.0, size=(n, pred_rows, S4)).astype(np.float32)   # speech enough to keep frames in the cache
    return E, P


def pct(v):
    v = np.sort(np.asarray(v) * 1e3)
    return float(np.percentile(v, 50)), float(np.percentile(v, 99))


def run(cfg, name, n, pushes, rng):
    sf = SortformerStreams(cfg)
    ids = np.array([sf.open() for _ in range(n)], np.int32)
    E, P = inputs(cfg, n, rng)
    warm = -(-(cfg.spkcache_len + cfg.fifo_len + cfg.spkcache_update_period) // cfg.chunk_len) + 2
    for w in range(warm):   # a session's first chunk has no left context (SortformerDiarizer.swift:553)
        sf.update(ids, E, P, emb_lengths=E.shape[1] - (0 if w else cfg.chunk_left_context))
    for extra in range(1, 6):   # stagger: session i is i % 6 chunks ahead
        sel = ids[ids % 6 >= extra]
        if sel.size:
            sf.update(sel, E[:sel.size], P[:sel.size])
    rows = E.shape[1]
    dE, dP = _lib.DeviceBuffer(E.nbytes), _lib.DeviceBuffer(P.nbytes)
    dE.upload(E)
    dP.upload(P)
    dc, dt = _lib.DeviceBuffer(4 * n * rows * S4), _lib.DeviceBuffer(4 * n * rows * S4)
    dsc = _lib.DeviceBuffer(4 * n * cfg.spkcache_len * D)
    dff = _lib.DeviceBuffer(4 * n * max(cfg.fifo_len, 1) * D)
    out = []
    for variant in ("device", "host"):
        upd, inp, launches = [], [], []
        reps = pushes if (variant == "device" or n <= 512) else max(5, pushes // 4)
        for r in range(reps + 3):
            before = _lib.kernel_launch_count()
            t0 = time.perf_counter()
            if variant == "device":
                sf.update_device(ids, dE, rows, dP, P.shape[1], dc, dt)
                _lib.synchronize()
            else:
                sf.update(ids, E, P)
            t1 = time.perf_counter()
            if variant == "device":
                sf.model_inputs_device(ids, dsc, dff)
                _lib.synchronize()
            else:
                sf.model_inputs(ids)
            t2 = time.perf_counter()
            if r >= 3:
                upd.append(t1 - t0)
                inp.append(t2 - t1)
                launches.append(_lib.kernel_launch_count() - before)
        u50, u99 = pct(upd)
        i50, i99 = pct(inp)
        t50, t99 = pct(np.array(upd) + np.array(inp))
        out.append(dict(preset=name, sessions=n, variant=variant, update_p50_ms=round(u50, 3),
                        update_p99_ms=round(u99, 3), inputs_p50_ms=round(i50, 3), inputs_p99_ms=round(i99, 3),
                        tick_p50_ms=round(t50, 3), tick_p99_ms=round(t99, 3),
                        audio_per_tick_ms=cfg.chunk_len * 80, launches_per_tick=int(np.median(launches)), pushes=reps))
    for b in (dE, dP, dc, dt, dsc, dff):
        b.free()
    sf.close_handle()
    return out


def oracle_row(cfg, rng):
    from oracle import oracle_sortformer as O
    n = 64
    sess = [O.Session(vars(cfg)) for _ in range(n)]
    E, P = inputs(cfg, 1, rng)
    warm = -(-(cfg.spkcache_len + cfg.fifo_len + cfg.spkcache_update_period) // cfg.chunk_len) + 2
    times = []
    for step in range(warm + 30):
        for i, s in enumerate(sess):
            if step == 0 and i % 6:
                continue   # stagger a little, as on the device
            lc = cfg.chunk_left_context if s.chunks else 0
            rows = lc + cfg.chunk_len + cfg.chunk_right_context
            L = s.lengths()
            pr = L.spkcache_length + L.fifo_length + rows
            t0 = time.perf_counter()
            s.update(E[0, -rows:], P[0, :pr], lc, cfg.chunk_right_context)
            if step >= warm:
                times.append(time.perf_counter() - t0)
    return float(np.mean(times)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=40)
    ap.add_argument("--sessions", default="1,64,512,4096")
    ap.add_argument("--presets", default="default,balancedV2")
    a = ap.parse_args()
    assert _lib.device_count() >= 1, "needs an H100"
    _lib.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    rng = np.random.default_rng(0)
    for name in a.presets.split(","):
        cfg = SortformerConfig.preset(name)
        per_session_ms = oracle_row(cfg, rng)
        for n in (int(x) for x in a.sessions.split(",")):
            for row in run(cfg, name, n, a.pushes, rng):
                print(json.dumps(row), flush=True)
            print(json.dumps(dict(preset=name, sessions=n, variant="oracle (1 thread, per-session updates)",
                                  update_ms=round(per_session_ms * n, 3), per_session_us=round(per_session_ms * 1e3, 2))),
                  flush=True)


if __name__ == "__main__":
    main()
