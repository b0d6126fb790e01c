"""Centroid linkage (``ahc_kernels.cu``) against the reference across every placement of the merge kernel (run with
``-m gpu``).

``Solver::linkage_device`` places a problem by ``plan_linkage`` in ``ahc_placement.h``: how much master state lives in
shared memory (level 3, 2, 1 or 0), whether every node vector stays resident in the worker CTAs' shared memory or is
streamed from HBM in up to 16 rounds per scan thread, and which pass of the float32 initial nearest-neighbour filter
runs.  The functions below restate those formulas (``tests/test_host_logic.py`` checks the restatement against the
compiled header), and every shape here is computed from them for the device's own SM count, one point either side of
each boundary.  Every dendrogram must equal the reference's bit for bit (the compiled reference under ``oracle/_ref``
where it was built, else the oracle's restatement), and must be a well-formed tree: every id below 2N - 1 is a child
exactly once and the cluster sizes telescope to N.  The launch count confirms the filter path (8 launches with the
filter, 10 when its candidate list overflows and the exact pass decides, 4 without it).

Cases too slow for a live reference run (the resident -> streamed flip at D = 220 and 256, and 16 streamed rounds at
the capacity N = W * 2 048) are compared with the SHA-256 of the reference's dendrogram from
``tests/golden/ahc_placements.json``; their N assume a 132-SM H100 and they are skipped on other SM counts.  The oracle
runs on CPU threads while the GPU works; the last test prints every case with its placement and the oracle's share.
"""
import hashlib
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200 import clustering as cl

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))

# ---- the placement, restated from ahc_placement.h ----------------------------------------------------------------
K_THREADS, K_ROUNDS = 128, 16
SMEM_CAP = 227 * 1024 - 2048
FILTER_MIN_N = 2048


def _up(b):
    return (b + 15) & ~15


def master_smem_bytes(N, level):
    b = _up(8 * N) + 2 * _up(2 * N) + _up(4 * ((2 * N - 1 + 31) >> 5))
    return b + (_up(4 * N) if level >= 2 else 0) + (_up(4 * N) if level >= 3 else 0)


def worker_fixed_smem(D):
    return 3 * 8 * ((D + 1) & ~1) + 2 * 8 * (K_THREADS // 32) + 64


def cap_slots(D):
    fixed = worker_fixed_smem(D)
    if fixed + 8 * D > SMEM_CAP:
        return 0
    return min(K_THREADS, (SMEM_CAP - fixed) // (8 * D))


def placement(N, D, W, force_global=False, force_stream=False, filter_min_n=FILTER_MIN_N):
    """plan_linkage: the fields of Placement, in its order"""
    p = dict(status=0, level=0, idx16=0, cap_slots=0, resident=0, workers=0, slots_per_cta=0, rounds=0, capacity=0,
             smem=0, filter=0, keep_tmin=0, filter_rows=0)
    Ns = (N + 31) & ~31
    if N <= 65535:
        for lvl in (1, 2, 3):
            if master_smem_bytes(N, lvl) <= SMEM_CAP:
                p["level"] = lvl
    if force_global:
        p["level"] = 0
    p["idx16"] = int(p["level"] >= 1)
    p["filter"] = int(0 < filter_min_n <= N)
    p["keep_tmin"] = int(N * ((N + 63) // 64) <= 16 << 20)
    p["filter_rows"] = int(p["keep_tmin"] and 8 * D * 4 <= 48 * 1024)
    cap = p["cap_slots"] = cap_slots(D)
    if cap == 0:
        p["status"] = 5
        return p
    p["resident"] = int(cap * W >= N and not force_stream)
    worker_smem = worker_fixed_smem(D)
    if p["resident"]:
        p["workers"] = min(W, max(1, -(-N // cap)))
        p["slots_per_cta"] = -(-N // p["workers"])
        p["rounds"] = 1
        worker_smem += 8 * D * p["slots_per_cta"]
    else:
        p["workers"] = max(1, min(W, -(-Ns // K_THREADS)))
        p["rounds"] = -(-Ns // (p["workers"] * K_THREADS))
        p["capacity"] = p["workers"] * K_THREADS * K_ROUNDS
        if p["capacity"] < Ns:
            p["status"] = 5
            return p
    p["smem"] = max(worker_smem, master_smem_bytes(N, p["level"]) if p["level"] else 0)
    return p


def batch_lanes(set_count, n_max, D, sms):
    """plan_batch_lanes: (lanes, worker_limit)"""
    lanes = max(1, min(set_count, 4))
    cap = cap_slots(D)
    need = -(-min(n_max, 2 ** 31 - 1) // cap) if cap else 0
    if 0 < need and need + 1 <= sms:
        lanes = max(1, min(lanes, sms // (need + 1)))
    ns_max = (n_max + 31) & ~31
    while lanes > 1 and max(1, sms // lanes - 1) * K_THREADS * K_ROUNDS < ns_max:
        lanes -= 1
    return lanes, (0 if lanes == 1 else max(1, sms // lanes - 1))


def level_limits():
    """largest N of master levels 3, 2 and 1"""
    out = []
    for lvl in (3, 2, 1):
        lo, hi = 2, 65535
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if master_smem_bytes(mid, lvl) <= SMEM_CAP else (lo, mid - 1)
        out.append(lo)
    return out


def d_limit():
    """largest D the merge kernel accepts"""
    D = 1
    while cap_slots(D + 1):
        D += 1
    return D


def expected_launches(p, overflow=False):
    """stage, the initial nearest-neighbour pass (exact: 2; filter: 6, + the exact 2 on overflow), merge"""
    return 1 + ((6 + (2 if overflow else 0)) if p["filter"] else 2) + 1


# ---- running and checking -----------------------------------------------------------------------------------------
SEEN = []            # one row per case for the report
ORACLE_SECONDS = []  # CPU time of every live oracle run
T_START = time.perf_counter()


@pytest.fixture(scope="module")
def sms(gpu_lib):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def well_formed(z, N):
    kids = np.sort(np.concatenate([z[:, 0], z[:, 1]]).astype(np.int64))
    return np.array_equal(kids, np.arange(2 * N - 2)) and z[-1, 3] == N and np.all(z[:, 0] < z[:, 1])


def _oracle_z(oracle, x):
    t0 = time.perf_counter()
    st, z = oracle.centroid_linkage(x, use_ref=oracle.ref_available())
    ORACLE_SECONDS.append(time.perf_counter() - t0)
    return st, z


def _row(label, N, D, p, seconds):
    pass2 = ("rows" if p["filter_rows"] else ("dense+tmin" if p["keep_tmin"] else "dense")) if p["filter"] else "-"
    SEEN.append((label, N, D, p["level"], p["resident"], p["workers"], p["rounds"], pass2, seconds))


def run_cases(oracle, W, cases):
    """cases: (label, x, overflow) -> GPU Z bit-identical to the oracle's, well formed, with the expected launches.  The
    oracle runs on a thread pool (ctypes releases the GIL) while the GPU works through the cases in order."""
    with ThreadPoolExecutor(max(1, min(len(cases), os.cpu_count() or 1))) as ex:
        want = [ex.submit(_oracle_z, oracle, x) for _, x, _ in cases]
        got = []
        for label, x, overflow in cases:
            N, D = x.shape
            p = placement(N, D, W)
            assert p["status"] == 0, (label, p)
            before = _lib.kernel_launch_count()
            t0 = time.perf_counter()
            st, z = cl.centroid_linkage(x)
            seconds = time.perf_counter() - t0
            launches = _lib.kernel_launch_count() - before
            _row(label, N, D, p, seconds)
            assert st == 0, (label, st)
            assert launches == expected_launches(p, overflow), (label, launches, p)
            assert well_formed(z, N), label
            got.append(z)
        for (label, x, _), f, z in zip(cases, want, got):
            st2, z2 = f.result()
            assert st2 == 0 and np.array_equal(z, z2), (label, x.shape)


def normal(seed, N, D):
    return np.random.default_rng(seed).standard_normal((N, D))


# ---- master levels, resident / streamed, streamed rounds ---------------------------------------------------------
def test_master_levels_at_every_boundary(gpu_lib, oracle, sms):
    W = sms - 1
    cases = []
    for lim in level_limits():
        for N in (lim, lim + 1):
            cases.append((f"level {placement(N, 4, W)['level']}", normal(N, N, 4), False))
    assert [placement(x.shape[0], 4, W)["level"] for _, x, _ in cases] == [3, 2, 2, 1, 1, 0]
    run_cases(oracle, W, cases)


def test_resident_to_streamed_and_streamed_rounds(gpu_lib, oracle, sms):
    W = sms - 1
    cases = []
    for D in (4, 1024, 2048, 4096, d_limit()):
        flip = cap_slots(D) * W
        for N in (flip, flip + 1):
            cases.append((f"flip D={D}", normal(N + D, N, D), False))
    for i, (_, x, _) in enumerate(cases):
        assert placement(*x.shape, W)["resident"] == (i % 2 == 0)
    # 2 rounds per scan thread, then 3 with a partial last round (also level 0 and the dense filter pass 2 without kept
    # bounds)
    two, three = cap_slots(4) * W + 1, 2 * K_THREADS * W + 1
    assert placement(two, 4, W)["rounds"] == 2 and placement(three, 4, W)["rounds"] == 3
    assert placement(three, 4, W)["level"] == 0 and not placement(three, 4, W)["keep_tmin"]
    cases.append(("3 rounds", normal(3, three, 4), False))
    run_cases(oracle, W, cases)


def _golden():
    with open(os.path.join(HERE, "golden", "ahc_placements.json")) as f:
        return json.load(f)["cases"]


def _golden_rows(oracle, case):
    """tests/golden/make_ahc_placement_golden.py inputs()"""
    if case["kind"] == "speakers":
        emb, _ = synth.speaker_embeddings(case["n"], case["d"], 8, seed=case["seed"])
        return oracle.l2_normalize_rows(emb.astype(np.float64))
    return np.random.default_rng(case["seed"]).standard_normal((case["n"], case["d"]))


def test_hashed_flips_and_the_capacity(gpu_lib, oracle, sms):
    """The D = 220 and D = 256 flips and 16 rounds at the capacity, against the reference's dendrogram hashes; one point
    past the capacity is refused before any launch."""
    W = sms - 1
    if W != 131:
        pytest.skip(f"the hashed shapes sit at the boundaries of 131 worker CTAs; this device has {sms} SMs")
    g = _golden()
    assert cap_slots(219) == 128 and cap_slots(220) == 127
    for name, case in sorted(g.items()):
        x = _golden_rows(oracle, case)
        N, D = x.shape
        p = placement(N, D, W)
        if name.startswith("d1_capacity"):
            assert N == W * K_THREADS * K_ROUNDS and p["rounds"] == K_ROUNDS and p["level"] == 0
        else:
            assert p["resident"] == name.split("_")[1].startswith("resident") and abs(N - cap_slots(D) * W) <= 1, name
        before = _lib.kernel_launch_count()
        t0 = time.perf_counter()
        st, z = cl.centroid_linkage(x)
        seconds = time.perf_counter() - t0
        launches = _lib.kernel_launch_count() - before
        _row(f"hash {name}", N, D, p, seconds)
        assert st == 0 and well_formed(z, N), name
        assert hashlib.sha256(z.tobytes()).hexdigest() == case["z_sha256"], name
        assert launches in (expected_launches(p), expected_launches(p, overflow=True)), (name, launches)
    # capacity + 1: FA_RUNTIME_ERROR (the pipeline maps it to identity labels), refused before the first launch
    N = W * K_THREADS * K_ROUNDS + 1
    assert placement(N, 1, W)["status"] == 5
    before = _lib.kernel_launch_count()
    st, _ = cl.centroid_linkage(np.random.default_rng(1).standard_normal((N, 1)))
    assert st == 5 and _lib.kernel_launch_count() == before


# ---- dimensions and the filter ---------------------------------------------------------------------------------------
def test_dimensions_and_the_dimension_limit(gpu_lib, oracle, sms):
    W = sms - 1
    cases = [(f"D={D}", normal(100 + D, 2048, D), False) for D in (1, 2, 3, 7, 8, 9, 15, 17, 31, 33)]
    assert all(placement(2048, D, W)["filter_rows"] for D in (1, 33))
    # pass 2: rows kernel while a row of 8 floats per D fits 48 KB, dense kernel past it
    assert placement(2048, 1536, W)["filter_rows"] and not placement(2048, 1537, W)["filter_rows"]
    cases += [(f"D={D}", normal(D, 2048, D), False) for D in (1536, 1537)]
    run_cases(oracle, W, cases)
    # D = 7 196 is the largest dimension (one target vector and one node vector per CTA): it was run above at the flip.
    # D = 7 197 is refused with FA_RUNTIME_ERROR before any launch, which the pipeline maps to identity labels.
    assert d_limit() == 7196 and placement(4, 7197, W)["status"] == 5
    before = _lib.kernel_launch_count()
    st, _ = cl.centroid_linkage(normal(7, 4, 7197))
    assert st == 5 and _lib.kernel_launch_count() == before


def test_filter_boundaries_and_candidate_overflow(gpu_lib, oracle, sms):
    W = sms - 1
    assert not placement(2047, 16, W)["filter"] and placement(2048, 16, W)["filter"]
    assert placement(32768, 4, W)["keep_tmin"] and not placement(32769, 4, W)["keep_tmin"]
    cases = [(f"filter N={N}", normal(N, N, D), False) for N, D in ((2047, 16), (2048, 16), (32768, 4), (32769, 4))]
    rng = np.random.default_rng(77)
    # every row with all its earlier copies as candidates: 16 x C(256, 2) = 522 240 pairs overflow the 64 N = 262 144
    # list, 32 x C(128, 2) = 260 096 (plus about one per group's first row) do not
    over = np.repeat(rng.standard_normal((16, 8)), 256, axis=0)[rng.permutation(4096)]
    under = np.repeat(rng.standard_normal((32, 8)), 128, axis=0)[rng.permutation(4096)]
    cases += [("overflow 16x256", over, True), ("no overflow 32x128", under, False)]
    run_cases(oracle, W, cases)


# ---- worker-limited batch lanes ---------------------------------------------------------------------------------------
def _batch(sizes, D, seed):
    embs, rhos, offs = [], [], [0]
    psi = None
    for i, n in enumerate(sizes):
        e, _ = synth.speaker_embeddings(n, D, 4, weights=(0.4, 0.3, 0.2, 0.1), seed=seed + i)
        r, p = synth.synthetic_plda(e)
        psi = p if psi is None else psi
        embs.append(e); rhos.append(r); offs.append(offs[-1] + n)
    return embs, rhos, offs, psi


def _batch_equals_one_by_one(sizes, D, seed, oracle=None):
    embs, rhos, offs, psi = _batch(sizes, D, seed)
    c = cl.OfflineClusterer(psi=psi)
    t0 = time.perf_counter()
    labels, _ = c.cluster_batch(np.concatenate(embs), np.concatenate(rhos), offs)
    seconds = time.perf_counter() - t0
    for i, n in enumerate(sizes):
        single = c.cluster(embs[i], rhos[i])
        assert np.array_equal(labels[offs[i]:offs[i + 1]], single.labels), (sizes, i)
        if oracle is not None and i == 0:
            assert single.info["training_count"] == n
            t1 = time.perf_counter()
            want = oracle.ahc_cluster(embs[i].astype(np.float64), 0.6, use_ref=oracle.ref_available())
            ORACLE_SECONDS.append(time.perf_counter() - t1)
            assert np.array_equal(single.initial, want)
    return seconds


def test_worker_limited_lanes_equal_one_by_one(gpu_lib, oracle, sms):
    """A set too large to be resident even on the whole GPU runs streamed in a lane of SMs / lanes - 1 workers."""
    sizes = [20000, 300, 300, 300]
    lanes, limit = batch_lanes(len(sizes), max(sizes), 4, sms)
    p = placement(20000, 4, limit)
    assert lanes == 4 and not p["resident"] and p["rounds"] > 1, (lanes, limit, p)
    seconds = _batch_equals_one_by_one(sizes, 4, 500, oracle)
    _row(f"batch lane x{lanes}", 20000, 4, p, seconds)


def test_set_past_the_four_lane_capacity_equals_one_by_one(gpu_lib, sms):
    """65 537 rows exceed the streamed capacity of four lanes (32 workers on 132 SMs: 65 536 slots); the lane count drops
    until the set fits its lane, and the batch equals one call per set."""
    sizes = [65537, 300, 300, 300]
    lanes, limit = batch_lanes(len(sizes), max(sizes), 4, sms)
    p = placement(65537, 4, limit if limit else sms - 1)
    assert p["status"] == 0 and not p["resident"], (lanes, limit, p)
    if sms == 132:
        assert lanes == 3 and max(1, sms // 4 - 1) * K_THREADS * K_ROUNDS < 65537
    seconds = _batch_equals_one_by_one(sizes, 4, 600)
    _row(f"batch lane x{lanes}", 65537, 4, p, seconds)


def test_report_placements():
    """last in the file: every case with its placement, and the live oracle's CPU share"""
    print(f"\n{'case':28s} {'N':>7s} {'D':>5s} lvl res workers rounds pass2      GPU s")
    for label, N, D, lvl, res, w, r, pass2, s in SEEN:
        print(f"{label:28s} {N:7d} {D:5d} {lvl:3d} {res:3d} {w:7d} {r:6d} {pass2:10s} {s:5.2f}")
    wall = time.perf_counter() - T_START
    print(f"oracle: {len(ORACLE_SECONDS)} runs, {sum(ORACLE_SECONDS):.1f} CPU-s on threads; file wall time {wall:.1f} s")
