"""Times the diarizer timelines on the GPU: one tick of S live sortformerDefault sessions, the timeline push alone and as
Sortformer update + timeline push, host and device variants, the offline batch (64 one-hour files in one push plus
finalize), and the CPU oracle's addChunk per session times S.

    python scripts/gpu_timeline.py [--pushes 40] [--sessions 1,64,512,4096]

A tick carries the default Sortformer chunk: 6 finalized and 7 tentative rows per session.  A push is timed on the host
clock around the call and, for the device variants, one device synchronisation; p50 and p99 over `--pushes` pushes
after warm-up.  "update + push" adds fa_sortformer_update[_device] of the same sessions (default preset, warmed through
its first compressions) and, for the device variant, the synchronisation between the two handles.  The oracle row is
the restatement's addChunk (C++, -O2, one thread, through ctypes) on 64 sessions, per session, times S.  The card's name
and power limit are read through NVML in the same process (queries only).  One JSON line per row.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib                                                               # noqa: E402
from fluidaudio_b200.diarizer_timeline import SEGMENT, DiarizerTimelineConfig, DiarizerTimelines   # noqa: E402
from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams                     # noqa: E402
from scripts.gpu_sortformer_streams import card, inputs, pct                                   # noqa: E402

D, S4, FIN, TEN = 512, 4, 6, 7


def preds(rng, rows):
    on = (rng.uniform(size=(rows // 8 + 1, S4)) < 0.35).repeat(8, 0)[:rows]
    return np.where(on, rng.uniform(0.5, 1.0, (rows, S4)), rng.uniform(0.0, 0.5, (rows, S4))).astype(np.float32)


def timed(fn, reps, sync):
    out = []
    for r in range(reps + 3):
        t0 = time.perf_counter()
        fn()
        if sync:
            _lib.synchronize()
        if r >= 3:
            out.append(time.perf_counter() - t0)
    return pct(out)


def tick_rows(n, pushes):
    rng = np.random.default_rng(n)
    tl = DiarizerTimelines(DiarizerTimelineConfig.sortformer_default(), TEN)
    ids = [tl.open_session() for _ in range(n)]
    fin, ten = preds(rng, n * FIN), preds(rng, n * TEN)
    fr, tr = np.full(n, FIN, np.int64), np.full(n, TEN, np.int64)
    bf, bt = tl.segment_bound(fr, tr)
    dF, dT = _lib.DeviceBuffer(fin.nbytes), _lib.DeviceBuffer(ten.nbytes)
    dF.upload(fin)
    dT.upload(ten)
    dfs, dts = _lib.DeviceBuffer(SEGMENT.itemsize * bf), _lib.DeviceBuffer(SEGMENT.itemsize * bt)
    dfc, dtc = _lib.DeviceBuffer(8 * n), _lib.DeviceBuffer(8 * n)
    rows = []
    p50, p99 = timed(lambda: tl.push_packed(ids, fin, fr, ten, tr), pushes, False)
    rows.append(dict(case="push", variant="host", sessions=n, p50_ms=p50, p99_ms=p99))
    p50, p99 = timed(lambda: tl.push_device(ids, dF, fr, dT, tr, dfs, dts, dfc, dtc), pushes, True)
    rows.append(dict(case="push", variant="device", sessions=n, p50_ms=p50, p99_ms=p99))

    # Sortformer update + timeline push
    cfg = SortformerConfig.preset("default")
    sf = SortformerStreams(cfg)
    sids = np.array([sf.open() for _ in range(n)], np.int32)
    E, P = inputs(sf.config, n, rng)
    warm = -(-(cfg.spkcache_len + cfg.fifo_len + cfg.spkcache_update_period) // cfg.chunk_len) + 2
    for w in range(warm):
        sf.update(sids, E, P, emb_lengths=E.shape[1] - (0 if w else cfg.chunk_left_context))
    dE, dP = _lib.DeviceBuffer(E.nbytes), _lib.DeviceBuffer(P.nbytes)
    dE.upload(E)
    dP.upload(P)
    dc, dt = _lib.DeviceBuffer(4 * n * E.shape[1] * S4), _lib.DeviceBuffer(4 * n * E.shape[1] * S4)

    def host_tick():
        conf, tent = sf.update(sids, E, P)
        tl.push(ids, conf, tent)

    def device_tick():
        cr, trr = sf.update_device(sids, dE, E.shape[1], dP, P.shape[1], dc, dt)
        _lib.synchronize()
        tl.push_device(ids, dc, cr, dt, trr, dfs, dts, dfc, dtc)

    reps = pushes if n <= 512 else max(5, pushes // 4)
    p50, p99 = timed(host_tick, reps, False)
    rows.append(dict(case="update+push", variant="host", sessions=n, p50_ms=p50, p99_ms=p99))
    p50, p99 = timed(device_tick, pushes, True)
    rows.append(dict(case="update+push", variant="device", sessions=n, p50_ms=p50, p99_ms=p99))
    for b in (dF, dT, dfs, dts, dfc, dtc, dE, dP, dc, dt):
        b.free()
    sf.close_handle()
    tl.close_handle()
    return rows


def offline_row(files=64, T=45000):
    rng = np.random.default_rng(1)
    cfg = DiarizerTimelineConfig.sortformer_default()
    cfg.max_stored_frames = T
    tl = DiarizerTimelines(cfg, 0)
    ids = [tl.open_session() for _ in range(files)]
    fin = preds(rng, files * T)
    fr, tr = np.full(files, T, np.int64), np.zeros(files, np.int64)
    bf, bt = tl.segment_bound(fr, tr)
    dF, dT = _lib.DeviceBuffer(fin.nbytes), _lib.DeviceBuffer(4)
    dF.upload(fin)
    dfs, dts = _lib.DeviceBuffer(SEGMENT.itemsize * bf), _lib.DeviceBuffer(SEGMENT.itemsize * max(bt, 1))
    dfc, dtc = _lib.DeviceBuffer(8 * files), _lib.DeviceBuffer(8 * files)

    def run():
        tl.reset(ids)
        tl.push_device(ids, dF, fr, dT, tr, dfs, dts, dfc, dtc)
        tl.finalize(ids)

    p50, p99 = timed(run, 10, True)
    for b in (dF, dT, dfs, dts, dfc, dtc):
        b.free()
    tl.close_handle()
    return dict(case="offline rebuild", variant="device", files=files, frames=T, p50_ms=p50, p99_ms=p99)


def oracle_per_session(pushes=40, n=64):
    from oracle import oracle_timeline as TL
    rng = np.random.default_rng(2)
    cfg = vars(DiarizerTimelineConfig.sortformer_default())
    refs = [TL.Timeline(cfg) for _ in range(n)]
    fin, ten = preds(rng, FIN), preds(rng, TEN)
    t0 = time.perf_counter()
    for _ in range(pushes):
        for r in refs:
            r.add_chunk(fin, ten)
    return (time.perf_counter() - t0) / (pushes * n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=40)
    ap.add_argument("--sessions", default="1,64,512,4096")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    _lib.set_device(0)
    where = card()
    per = oracle_per_session()
    lines = []
    for n in (int(s) for s in a.sessions.split(",")):
        for r in tick_rows(n, a.pushes):
            lines.append(r)
        lines.append(dict(case="oracle addChunk x S", variant="cpu", sessions=n, ms=per * n * 1e3))
    lines.append(offline_row())
    for r in lines:
        r["card"] = where
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
