"""Dendrogram hashes for the centroid-linkage placement sweep cases too slow for a live oracle run
(tests/test_gpu_ahc_sweep.py).

Run where the reference sources exist, so that oracle/_ref/liboracle_fc.so is built:

    python tests/golden/make_ahc_placement_golden.py

Each case's input is regenerated from its seed by ``inputs`` below (the sweep imports the same function), run through the
UNMODIFIED reference FastClusterWrapper.cpp, and stored as the SHA-256 of the Z bytes.  The dendrogram does not depend
on where the GPU places the problem, so the hashes hold on any GPU; the N of the capacity case is the merge kernel's
streamed capacity W * 2 048 for W = 131 worker CTAs (a 132-SM H100 SXM).
  * d220_*, d256_*: both sides of the resident -> streamed flip at the first D that holds fewer than 128 node vectors
    per CTA (cap(220) = 127, 127 * 131 = 16 637) and at D = 256 (cap = 109, 109 * 131 = 14 279), normalised synthetic
    speaker embeddings.
  * d1_capacity_268288: D = 1 at the largest N the merge kernel accepts on 131 workers: 16 streamed rounds per thread.
"""
import hashlib
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

CASES = {
    "d220_resident_16637": {"kind": "speakers", "seed": 16637, "n": 16637, "d": 220},
    "d220_streamed_16638": {"kind": "speakers", "seed": 16638, "n": 16638, "d": 220},
    "d256_resident_14279": {"kind": "speakers", "seed": 14279, "n": 14279, "d": 256},
    "d256_streamed_14280": {"kind": "speakers", "seed": 14280, "n": 14280, "d": 256},
    "d1_capacity_268288": {"kind": "normal", "seed": 268288, "n": 131 * 2048, "d": 1},
}


def inputs(case: dict) -> np.ndarray:
    """The rows a case hashes: normalised synthetic speaker embeddings, or standard normal rows."""
    from fluidaudio_b200 import synth
    from oracle import oracle as O
    if case["kind"] == "speakers":
        emb, _ = synth.speaker_embeddings(case["n"], case["d"], 8, seed=case["seed"])
        return O.l2_normalize_rows(emb.astype(np.float64))
    return np.random.default_rng(case["seed"]).standard_normal((case["n"], case["d"]))


def one(name: str) -> tuple:
    from oracle import oracle as O
    case = CASES[name]
    x = inputs(case)
    t0 = time.perf_counter()
    st, z = O.centroid_linkage(x, use_ref=True)
    seconds = time.perf_counter() - t0
    assert st == 0, (name, st)
    return name, dict(case, z_sha256=hashlib.sha256(z.tobytes()).hexdigest(), reference_seconds=round(seconds, 1))


def main():
    from oracle import oracle as O
    O.build()
    assert O.ref_available(), "oracle/_ref/liboracle_fc.so missing: run `make -C oracle ref` where the reference sources are"
    with ProcessPoolExecutor(len(CASES)) as ex:
        rows = dict(ex.map(one, sorted(CASES)))
    out = {"linkage": "unmodified reference FastClusterWrapper.cpp (oracle/_ref), one CPU core per case",
           "cases": rows}
    with open(os.path.join(HERE, "ahc_placements.json"), "w") as f:
        json.dump(out, f, indent=1)
    for name, r in rows.items():
        print(f"{name}: {r['z_sha256']} ({r['reference_seconds']} s)")


if __name__ == "__main__":
    main()
