"""Times CTC decoding on the GPU: beam search (B = 100, K = 40) over 1 000 clips of 188 frames (15 s at 80 ms) x 1025
columns without and with a synthetic bigram LM of 20 000 words and 100 000 bigrams, over one hour (45 000 frames), and
greedy decoding of both workloads, beside the C++ oracle on one core.

    python scripts/gpu_ctc_decode_timing.py [--reps 10] [--oracle-clips 3] [--out rows.jsonl]

Every call is timed on the host clock around the call, which includes its synchronisation, with the log-probs and
the ids in HBM (the _device variants), p50 and p99 over `--reps` calls after two warm-up calls.  The oracle arm decodes
the first `--oracle-clips` clips (for the hour, its first `--oracle-clips` x 188 frames) one after another on one core
and scales to the whole workload; its row says so.  The card's name and power limit are read through NVML in the same
process (queries only).  One JSON line per row on stdout, and in `--out` when given.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from fluidaudio_b200 import _lib                     # noqa: E402
from fluidaudio_b200 import ctc_decoding as D        # noqa: E402
from fluidaudio_b200 import ctc_spotting as S        # noqa: E402
from oracle import oracle_ctc_decode as O            # noqa: E402
import ctc_decode_cases as cases                     # noqa: E402

V, BLANK, CLIP = 1025, 1024, 188


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
        ts.append(time.perf_counter() - t0)
    a = np.asarray(ts) * 1e3
    return float(np.percentile(a, 50)), float(np.percentile(a, 99))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--oracle-clips", type=int, default=3)
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

    voc = cases.vocabulary(rng, V)
    pieces = cases.pieces(voc, V)
    uni, bi = cases.synthetic_lm(rng, words=20000, bigrams=100000, max_len=5)
    arpa = D.ARPALanguageModel()
    arpa.unigrams = {w: D.ARPALanguageModel.Entry(*e) for w, e in uni.items()}
    arpa.bigrams = {c: {w: D.ARPALanguageModel.Entry(p, np.float32(0)) for w, p in r.items()} for c, r in bi.items()}
    lm, lm_arrays = arpa.to_device(), O.LmArrays(uni, bi)
    dec = D.CtcDecoder(voc, V, BLANK)
    L = _lib.load()
    workloads = {"1000 clips x 188x1025": [CLIP] * 1000, "one hour 45000x1025": [45000]}
    for name, lens in workloads.items():
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        rows_n = int(off[-1])
        lp = S.apply_log_softmax(rng.normal(0, 3, size=(rows_n, V)).astype(np.float32), BLANK)
        d_lp, d_tok = _lib.DeviceBuffer(lp.nbytes), _lib.DeviceBuffer(4 * rows_n)
        d_lp.upload(lp)
        for with_lm in (False, True):
            model = lm if with_lm else None
            st, _, _, total = dec.beam_search_device(d_lp, off, d_tok, rows_n, model, 100, 0.3, 0.0, 40)
            p50, p99 = timed(lambda: dec.beam_search_device(d_lp, off, d_tok, rows_n, model, 100, 0.3, 0.0, 40), a.reps)
            n = a.oracle_clips
            t0 = time.perf_counter()
            for c in range(n):
                O.beam_search(lp[c * CLIP:(c + 1) * CLIP], pieces, lm_arrays if with_lm else None, 100, 0.3, 0.0, BLANK, 40)
            cpu = (time.perf_counter() - t0) * 1e3 * rows_n / (n * CLIP)
            emit(workload=f"beam B=100 K=40 {name}" + (" with LM" if with_lm else ""), ids=total, gpu_p50_ms=p50,
                 gpu_p99_ms=p99, oracle_one_core_ms=cpu,
                 oracle_note=f"timed over {n} x {CLIP} frames, scaled to {rows_n} frames")
        lengths, total = np.zeros(len(lens), np.int64), C.c_int64()

        def greedy():
            _lib.check(L.fa_ctc_greedy_device(d_lp.ptr, _lib.ptr(off), len(lens), V, BLANK, _lib.ptr(lengths),
                                              d_tok.ptr, rows_n, C.byref(total)), "fa_ctc_greedy_device")
        p50, p99 = timed(greedy, a.reps)
        emit(workload=f"greedy {name}", ids=int(total.value), gpu_p50_ms=p50, gpu_p99_ms=p99)
        d_lp.free()
        d_tok.free()
    dec.close()
    lm.close()
    if a.out:
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
