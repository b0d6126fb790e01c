"""Times streaming speaker tracking on the GPU: one 10 s tick (fa_od_embedding_inputs + fa_od_advance, logits and
embeddings fixed) at S = 1 / 64 / 512 / 4 096 sessions with 4 / 16 / 64 known speakers each, with host and device
buffers, beside the C++ oracle running the same sessions one after another on one host core.

    python scripts/gpu_online_diar_timing.py [--reps 30] [--out rows.jsonl]

Every call is timed on the host clock around the C calls, which end in a synchronisation (fa_od_advance waits for the
pushed sessions' headers), p50 and p99 over `--reps` ticks after two warm-up ticks.  The models are left out.  Each
session's embeddings are its own known speakers plus noise, so the databases keep their size while timed.  The oracle
arm calls oracle_od_chunk once per session through ctypes (a few microseconds of call overhead each) and is timed over
fewer ticks at large S.  The card's name and power limit are read through NVML in the same process (queries only).
One JSON line per row on stdout, and in `--out` when given.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fluidaudio_b200 import _lib                       # noqa: E402
from fluidaudio_b200 import online_diarizer as OD      # noqa: E402
from oracle import oracle_online_diar as O             # noqa: E402

F, D = 589, 256


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
        return name.value.decode(), mw.value / 1000.0
    except Exception:
        return "unknown", None


def stats(ts):
    ts = np.sort(np.asarray(ts) * 1e3)
    return float(np.percentile(ts, 50)), float(np.percentile(ts, 99))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, watts = card()
    out = open(a.out, "w") if a.out else None
    L = _lib.load()
    rng = np.random.default_rng(0)
    for S in (1, 64, 512, 4096):
        for K in (4, 16, 64):
            dbs = OD.SpeakerDatabases(F)
            sids = [dbs.open() for _ in range(S)]
            voices = rng.normal(size=(K, D)).astype(np.float32)
            for s in sids:
                dbs.initialize_known_speakers(s, [OD.Speaker(str(k + 1), voices[k], 5.0) for k in range(K)])
            lg = np.zeros((S, F, 7), np.float32)
            lg[:, np.arange(F), (np.arange(F) // 100) % 4] = 4.0
            emb = (voices[rng.integers(0, K, size=(S, 3))] + rng.normal(0, 0.05, (S, 3, D))).astype(np.float32)
            cfg = dbs.config.c()
            s32 = np.ascontiguousarray(sids, np.int32)
            offs = np.zeros(S, np.float64)
            bound = 3 * ((F + 1) // 2)
            masks, need = np.empty((S, 3, F), np.float32), np.empty((S, 3), np.int32)
            asg, cnt = np.empty((S, 3, 2), np.int64), np.empty(S, np.int32)
            ids, vals = np.empty((S, bound, 2), np.int64), np.empty((S, bound, 3), np.float32)
            dev = {k: _lib.DeviceBuffer(v) for k, v in dict(lg=lg.nbytes, m=masks.nbytes, n=need.nbytes, e=emb.nbytes,
                                                           a=asg.nbytes, c=cnt.nbytes, i=ids.nbytes,
                                                           v=vals.nbytes).items()}
            dev["lg"].upload(lg)
            dev["e"].upload(emb)

            def tick_host():
                _lib.check(L.fa_od_embedding_inputs(dbs._h, S, s32.ctypes.data, lg.ctypes.data, C.byref(cfg),
                                                    masks.ctypes.data, need.ctypes.data), "inputs")
                _lib.check(L.fa_od_advance(dbs._h, S, s32.ctypes.data, emb.ctypes.data, offs.ctypes.data,
                                           C.byref(cfg), asg.ctypes.data, cnt.ctypes.data, ids.ctypes.data,
                                           vals.ctypes.data), "advance")

            def tick_device():
                _lib.check(L.fa_od_embedding_inputs_device(dbs._h, S, s32.ctypes.data, dev["lg"].ptr, C.byref(cfg),
                                                           dev["m"].ptr, dev["n"].ptr), "inputs")
                _lib.check(L.fa_od_advance_device(dbs._h, S, s32.ctypes.data, dev["e"].ptr, offs.ctypes.data,
                                                  C.byref(cfg), dev["a"].ptr, dev["c"].ptr, dev["i"].ptr,
                                                  dev["v"].ptr), "advance")

            row = {"sessions": S, "speakers": K, "card": name, "power_limit_w": watts}
            for label, fn in (("host", tick_host), ("device", tick_device)):
                fn(), fn()
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    fn()
                    ts.append(time.perf_counter() - t0)
                row[f"{label}_p50_ms"], row[f"{label}_p99_ms"] = stats(ts)
            refs = [O.Session() for _ in sids]
            sp = np.zeros(K, O.SPEAKER)
            sp["key"] = sp["numeric"] = np.arange(1, K + 1)
            sp["has_numeric"] = sp["update_count"] = 1
            sp["duration"] = 5.0
            for r in refs:
                r.initialize(sp, voices, np.zeros((0, D), np.float32), 3)
            res = O.resolved()
            oreps = max(3, min(a.reps, 2000 // S))
            ts = []
            for _ in range(oreps):
                t0 = time.perf_counter()
                for j, r in enumerate(refs):
                    r.chunk(lg[j], 160000, emb[j], 0.0, res)
                ts.append(time.perf_counter() - t0)
            row["oracle_p50_ms"], row["oracle_p99_ms"] = stats(ts)
            row["oracle_ticks"] = oreps
            for b in dev.values():
                b.free()
            dbs.close_handle()
            line = json.dumps(row)
            print(line, flush=True)
            if out:
                out.write(line + "\n")


if __name__ == "__main__":
    main()
