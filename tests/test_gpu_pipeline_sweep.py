"""The clustering pipeline (``cluster_pipeline`` in ``cluster_pipeline.cu``) and its batch entry points on every branch (run with
``-m gpu``).

The C ABI is called through ctypes, so NULL outputs, ``max_centroids`` and ``init_smoothing`` are reachable.  Every case
is checked twice:

1. against the oracle (``oracle.diarize_cluster`` with the compiled reference AHC where it was built): ``initial`` on the
   training rows and -1 on filtered rows, every non-timing ``info`` field and the labels exactly; centroids within 1e-9
   with the same NaN / Inf footprint.  Cases that are degenerate by construction (identity init, threshold 0, duplicate
   or zero rows, one-dimensional embeddings) compare labels only where the oracle's top two scores differ by more than
   1e-9, and the undecided rows must be a small minority;
2. against the library's own standalone entry points, bit for bit: ``fa_ahc_cluster``, ``fa_vbx_refine``,
   ``fa_compute_centroids`` (or ``fa_kmeans_cluster`` when a speaker count re-clusters), ``fa_assign_embeddings`` and
   ``fa_constrained_assign`` on the same training rows give the pipeline's labels, ``initial``, ``info`` and centroid
   bytes.  The GPU is deterministic and the kernels are the same, so any difference is a glue defect (a wrong gather
   index or widen, two centroid normalisations that disagree in the last bit).

Each case names the branch it must take, and the launch-count delta (``pipeline_launches`` below) confirms it:

| Branch of ``cluster_pipeline`` | Entered by | Proof |
|---|---|---|
| every row finite: no gather | ``plain``, the shape and config cases | training_count == N; no gather launches |
| filtered rows: two gathers | ``nan_first_row``, ``nan_last_row``, ``nan_last_element``, ``inf_rows``, ``nan_emb_chunks`` | training_count < N, initial -1 there; +2 launches |
| no finite row: every row trains | ``all_nonfinite`` | training_count == N; AHC stops after its exact nearest-neighbour pass (3 launches) |
| one training row: no AHC | ``one_finite``, ``n1`` | initial_clusters 1; no normalise / AHC launches |
| AHC on two rows | ``two_finite``, ``n2`` | training_count 2; normalise + 4 AHC launches |
| AHC succeeds, dendrogram cut | every other case | initial equals the reference's |
| AHC reports NaN -> identity labels | ``all_nonfinite`` | initial_clusters == N |
| AHC refuses D >= 7 197 -> identity labels | ``wide_7197`` | initial_clusters == training_count; normalise only, no AHC launch |
| AHC refuses N past the merge kernel's capacity -> identity, then VBx needs Tn^2 doubles | ``test_past_the_merge_capacity...`` | FA_ALLOCATION_FAILURE after 3 launches (widen, finite rows, normalise) |
| fused VBx (S <= 64) / staged VBx and centroids (S > 64) | ``plain`` / ``threshold_0`` | the VBx and centroid launch formulas |
| speaker count satisfied | ``min_speakers_1`` | was_adjusted 0 |
| speaker count violated -> K-Means + normalisation | ``num_speakers_1_chunks`` | was_adjusted 1; K-Means launches + 1 |
| non-finite rho in a training row | ``rho_nan``, ``rho_nan_chunks`` | every E-step row falls back to uniform gamma: S identical centroids, every score tied, label 0 |
| no speaker with pi > 1e-7 -> one-hot recompute | removed: unreachable, see Proof | VBx renormalises pi to sum 1 and falls back to 1/S when the sum is not finite, so some pi >= 1/S > 1e-7 for any S an arena can hold |
| K == 0 after that -> mean of all rows | removed: unreachable, see Proof | the one-hot recompute would give pi = 1 to all S >= 1 speakers, and K-Means returns min(target, Tn) >= 1 rows; the pipeline reports K == 0 as an internal FA_RUNTIME_ERROR |
| constrained assignment (chunks, K > 1, not adjusted) | ``nan_emb_chunks``, ``chunk_overflow``, ``rho_nan_chunks`` | labels equal ``fa_constrained_assign``; -2 where a chunk has more local speakers than clusters |
| chunks with K == 1, or adjusted -> plain argmax | ``k1_chunks``, ``num_speakers_1_chunks`` | no -2 label |
| NULL initial / centroids / info, max_centroids | ``test_null_outputs...``, ``test_max_centroids...`` | same labels; the first min(K, max) rows byte-equal, the rest untouched |

The last test prints the worst centroid deviation from the oracle as a fraction of 1e-9 and the file's wall time.
"""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth

pytestmark = pytest.mark.gpu

NO = _lib.NO_VALUE
K_ETHREADS, K_FUSED_MAX_S, SMEM = 128, 64, 200 * 1024   # vbx_kernels.cu
FILTER_MIN_N = 2048                                       # ahc_kernels.cu: the float32 filter from N = 2048
D_REFUSED = 7197                                          # ahc_placement.h: the first D the merge kernel refuses
SENTINEL = -1234.5678
INFO_FIELDS = ("training_count", "initial_clusters", "vbx_iterations", "centroid_count", "was_adjusted",
               "detected_clusters")
WORST = [0.0]   # worst |centroid - oracle| seen, over 1e-9
T_START = time.perf_counter()


# ---- launch counts (tests/test_launch_counts.py, extended with AHC's NaN stop and the identity fallback) ------------
def vbx_launches(S, D, max_it):
    fused = S <= K_FUSED_MAX_S and 8 * (S * D + 2 * S + K_ETHREADS * S + K_ETHREADS) <= SMEM
    if fused:
        return 3 if max_it == 0 else 2 * max_it + 4
    return 4 * max_it + 2


def centroid_launches(S):
    return 3 if S <= K_FUSED_MAX_S else 2


def ahc_launches(N, ahc):
    """linkage_device: stage + initial nearest-neighbour pass + merge; "nan" stops after the exact pass, "refused"
    (D or N past the merge kernel's limits) launches nothing"""
    nn = 6 if N >= FILTER_MIN_N else 2
    return {"ok": 1 + nn + 1, "nan": 1 + nn + (2 if N >= FILTER_MIN_N else 0), "refused": 0}[ahc]


def pipeline_launches(N, info, R, max_it, ahc="ok", kmeans=None):
    """widen + finite rows, two gathers when rows were filtered, normalise + AHC from two training rows, VBx, then the
    centroids or K-Means + normalisation, assignment"""
    Tn, S = info["training_count"], info["initial_clusters"]
    n = 2 + (2 if Tn != N else 0)
    if Tn >= 2:
        n += 1 + ahc_launches(Tn, ahc)
    n += vbx_launches(S, R, max_it)
    if kmeans is not None:
        n += kmeans + 1
    else:
        n += centroid_launches(S)
    return n + 1


# ---- calling the C ABI --------------------------------------------------------------------------------------------
def config(threshold=0.6, Fa=0.07, Fb=0.8, max_iterations=20, epsilon=1e-4, init_smoothing=7.0, num_speakers=NO,
           min_speakers=NO, max_speakers=NO):
    cfg = _lib.ClusterConfig()   # every field set here: the cases are built at import, without loading the library
    cfg.threshold = threshold
    cfg.vbx.Fa, cfg.vbx.Fb, cfg.vbx.max_iterations = Fa, Fb, max_iterations
    cfg.vbx.epsilon, cfg.vbx.init_smoothing = epsilon, init_smoothing
    cfg.num_speakers, cfg.min_speakers, cfg.max_speakers = num_speakers, min_speakers, max_speakers
    return cfg


def info_dict(info):
    return {f: int(getattr(info, f)) for f in INFO_FIELDS}


def pipeline(case, want_initial=True, want_centroids=True, want_info=True, max_centroids=None):
    """one fa_diarize_cluster(_chunks) call: (status, labels, initial, centroid buffer, info, launches)"""
    L = _lib.load()
    emb, rho, psi, cfg, chunk = case["emb"], case["rho"], case["psi"], case["cfg"], case["chunk"]
    N, E = emb.shape
    R = rho.shape[1]
    mc = N if max_centroids is None else max_centroids
    labels = np.full(N, -7, np.int32)
    initial = np.full(N, -7, np.int32) if want_initial else None
    cent = np.full((max(mc, 1), E), SENTINEL) if want_centroids else None
    info = _lib.ClusterInfo()
    args = (emb.ctypes.data, rho.ctypes.data, N, E, R, _lib.ptr(psi), C.byref(cfg))
    outs = (labels.ctypes.data, _lib.ptr(initial), _lib.ptr(cent), mc, C.byref(info) if want_info else None)
    before = L.fa_kernel_launch_count()
    if chunk is None:
        st = L.fa_diarize_cluster(*args, *outs)
    else:
        st = L.fa_diarize_cluster_chunks(*args, chunk.ctypes.data, *outs)
    launches = L.fa_kernel_launch_count() - before
    err = L.fa_last_error().decode("utf-8", "replace") if st else ""
    return dict(status=int(st), error=err, labels=labels, initial=initial, centroids=cent,
                info=info_dict(info) if want_info else None, launches=launches)


def _ok(st, where):
    _lib.check(st, where)


def compose(case):
    """The pipeline restated as the library's standalone entry points on the same training rows."""
    L = _lib.load()
    emb, rho, psi, cfg, chunk = case["emb"], case["rho"], case["psi"], case["cfg"], case["chunk"]
    N, E = emb.shape
    R = rho.shape[1]
    feats = emb.astype(np.float64)
    idx = np.nonzero(np.isfinite(emb).all(axis=1))[0]
    if idx.size == 0:
        idx = np.arange(N)
    train, trho, Tn = np.ascontiguousarray(feats[idx]), np.ascontiguousarray(rho[idx]), idx.size
    init = np.zeros(Tn, np.int32)
    if Tn >= 2:
        _ok(L.fa_ahc_cluster(train.ctypes.data, Tn, E, cfg.threshold, init.ctypes.data), "fa_ahc_cluster")
    S = int(init.max()) + 1
    cap = max(cfg.vbx.max_iterations, 1)
    gamma, pi, elbos = np.zeros((Tn, S)), np.zeros(S), np.zeros(cap)
    hard, its = np.zeros(Tn, np.int32), C.c_int32()
    _ok(L.fa_vbx_refine(trho.ctypes.data, Tn, R, _lib.ptr(psi), 0 if psi is None else psi.size, init.ctypes.data, S,
                        C.byref(cfg.vbx), gamma.ctypes.data, pi.ctypes.data, elbos.ctypes.data, hard.ctypes.data,
                        C.byref(its)), "fa_vbx_refine")
    detected = len({h for h in hard.tolist() if 0 <= h < S})
    adjusted, km_launches = False, None
    if (cfg.num_speakers, cfg.min_speakers, cfg.max_speakers) != (NO, NO, NO):
        lo, hi = C.c_int64(), C.c_int64()
        _ok(L.fa_speaker_constraints_resolve(Tn, cfg.num_speakers, cfg.min_speakers, cfg.max_speakers, C.byref(lo),
                                             C.byref(hi)), "resolve")
        if detected < lo.value or detected > hi.value:
            target = lo.value if detected < lo.value else hi.value
            cents, lab = np.zeros((target, E)), np.zeros(Tn, np.int32)
            rows, best = C.c_int32(), C.c_int32()
            before = L.fa_kernel_launch_count()
            _ok(L.fa_kmeans_cluster(train.ctypes.data, Tn, E, target, 100, 10, 0, lab.ctypes.data, cents.ctypes.data,
                                    target, C.byref(rows), C.byref(best)), "fa_kmeans_cluster")
            km_launches = L.fa_kernel_launch_count() - before
            cents, adjusted = cents[:rows.value].copy(), True

    def centroids(g, p):
        out, K = np.zeros((S, E)), C.c_int32()
        _ok(L.fa_compute_centroids(train.ctypes.data, Tn, E, g.ctypes.data, p.ctypes.data, S, out.ctypes.data,
                                   C.byref(K)), "fa_compute_centroids")
        return out[:K.value].copy()

    if not adjusted:
        cents = centroids(gamma, pi)
    K = cents.shape[0]
    assert K > 0, "no speaker with pi > 1e-7"   # an internal error in the pipeline, unreachable (module docstring)
    labels, scores = np.zeros(N, np.int32), np.zeros((N, max(K, 1)))
    _ok(L.fa_assign_embeddings(feats.ctypes.data, N, E, cents.ctypes.data, K, labels.ctypes.data, scores.ctypes.data),
        "fa_assign_embeddings")
    if chunk is not None and K > 1 and not adjusted:
        _ok(L.fa_constrained_assign(scores.ctypes.data, N, K, chunk.ctypes.data, labels.ctypes.data), "constrained")
    initial = np.full(N, -1, np.int32)
    initial[idx] = init
    info = dict(training_count=Tn, initial_clusters=S, vbx_iterations=its.value, centroid_count=K,
                was_adjusted=int(adjusted), detected_clusters=detected)
    return dict(labels=labels, initial=initial, centroids=cents, info=info, kmeans=km_launches)


def opt(v):
    return None if v == NO else int(v)


def check_oracle(oracle, case, run):
    emb, rho, psi, cfg, chunk = case["emb"], case["rho"], case["psi"], case["cfg"], case["chunk"]
    v = cfg.vbx
    o = oracle.diarize_cluster(emb, rho, np.ones(rho.shape[1]) if psi is None else psi, threshold=cfg.threshold,
                               Fa=v.Fa, Fb=v.Fb, max_iterations=v.max_iterations, epsilon=v.epsilon,
                               use_ref=oracle.ref_available(), chunk_indices=chunk, num_speakers=opt(cfg.num_speakers),
                               min_speakers=opt(cfg.min_speakers), max_speakers=opt(cfg.max_speakers),
                               init_smoothing=v.init_smoothing, initial=case.get("oracle_initial"))
    name, N = case["name"], emb.shape[0]
    idx = o.training_indices
    filtered = np.ones(N, bool)
    filtered[idx] = False
    assert np.array_equal(run["initial"][idx], o.initial), name
    assert (run["initial"][filtered] == -1).all(), name
    want = dict(training_count=idx.size, initial_clusters=max(1, len(set(o.initial.tolist()))),
                vbx_iterations=o.vbx.elbos.size,
                centroid_count=o.centroids.shape[0], was_adjusted=int(o.was_adjusted),
                detected_clusters=o.detected_clusters)
    assert run["info"] == want, (name, run["info"], want)
    K = o.centroids.shape[0]
    got = run["centroids"][:K]
    for test in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(test(got), test(o.centroids)), (name, test.__name__)
    fin = np.isfinite(o.centroids)
    dev = float(np.abs(got[fin] - o.centroids[fin]).max()) if fin.any() else 0.0
    WORST[0] = max(WORST[0], dev / 1e-9)
    assert dev <= 1e-9, (name, dev)
    if not case["degenerate"]:
        assert np.array_equal(run["labels"], o.labels), (name, np.nonzero(run["labels"] != o.labels)[0][:10])
        return o
    # degenerate by construction: labels where the oracle's top two scores differ by more than 1e-9
    ok = np.isfinite(emb).all(axis=1)
    cn = o.centroids / np.maximum(np.linalg.norm(o.centroids, axis=1, keepdims=True), 1e-300)
    e = np.where(ok[:, None], emb, 0.0).astype(np.float64)
    sc = (e / np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-300)) @ cn.T
    srt = np.sort(sc, axis=1)
    decided = ok & ((srt[:, -1] - srt[:, -2] > 1e-9) if K > 1 else np.ones(N, bool))
    if chunk is not None:   # a tie anywhere in a chunk can move the chunk's matching
        decided &= np.isin(chunk, np.unique(chunk[~decided]), invert=True)
    assert np.array_equal(run["labels"][decided], o.labels[decided]), name
    assert (~decided).sum() <= max(2, N // 10), (name, int((~decided).sum()))
    return o


def check_composition(case, run, comp):
    name = case["name"]
    assert np.array_equal(run["labels"], comp["labels"]), (name, np.nonzero(run["labels"] != comp["labels"])[0][:10])
    assert np.array_equal(run["initial"], comp["initial"]), name
    assert run["info"] == comp["info"], (name, run["info"], comp["info"])
    K = comp["info"]["centroid_count"]
    assert run["centroids"][:K].tobytes() == comp["centroids"].tobytes(), name


# ---- fixtures -----------------------------------------------------------------------------------------------------
def blobs(n, d, k, seed):
    """k well separated speakers; the noise per dimension shrinks above 64 dimensions so that its norm stays put"""
    return synth.speaker_embeddings(n, d, k, sigma=0.02 * min(1.0, (64 / d) ** 0.5), seed=seed)[0]


def plda(emb, R, seed=5):
    """rho [n x R] from the embeddings through a random projection (R may exceed the embedding width), plus a little
    independent noise; psi positive.  At this scale VBx keeps the speakers apart, so every label is decisive."""
    e = np.nan_to_num(emb.astype(np.float64), nan=0.0, posinf=0.0, neginf=0.0)
    rng = np.random.default_rng(seed)
    unit = e / np.maximum(np.linalg.norm(e, axis=1, keepdims=True), 1e-30)
    W = 4.0 * rng.standard_normal((e.shape[1], R)) * np.sqrt(R / e.shape[1])
    rho = (unit - unit.mean(axis=0, keepdims=True)) @ W + 0.05 * rng.standard_normal((e.shape[0], R))
    psi = 0.1 + 10.0 * np.exp(-np.arange(R) / 32.0)
    return np.ascontiguousarray(rho), psi


def make(name, emb, R=32, cfg=None, chunk=None, psi=True, degenerate=False, ahc="ok", adjusted=False, rho=None,
         oracle_initial=None):
    r, p = plda(emb, R)
    return dict(name=name, emb=np.ascontiguousarray(emb, np.float32), rho=r if rho is None else rho,
                psi=p if psi else None, cfg=cfg or config(), chunk=chunk, degenerate=degenerate, ahc=ahc,
                adjusted=adjusted, oracle_initial=oracle_initial)


def chunks_of(n, per=2):
    return (np.arange(n) // per).astype(np.int32)


def _with(emb, rows, value, col=None):
    e = emb.copy()
    if col is None:
        e[rows] = value
    else:
        e[rows, col] = value
    return e


def build_cases():
    base = blobs(300, 64, 4, 1)
    cases = [make("plain", base)]
    # training subset
    cases += [make("nan_first_row", _with(base, 0, np.nan)), make("nan_last_row", _with(base, -1, np.nan)),
              make("nan_last_element", _with(base, 5, np.nan, col=-1))]
    e = _with(base, 7, np.inf, col=3)
    cases.append(make("inf_rows", _with(e, 100, -np.inf, col=0)))
    small = blobs(40, 64, 3, 2)
    one = np.full_like(small, np.nan)
    one[17] = small[17]
    two = np.full_like(small, np.nan)
    two[[3, 31]] = small[[3, 31]]
    cases += [make("one_finite", one), make("two_finite", two),
              make("all_nonfinite", np.full_like(small, np.nan), ahc="nan")]   # every score NaN: all labels 0
    dup = base.copy()
    dup[[3, 4]] = 0.0
    dup[10:20] = dup[9]
    cases.append(make("zero_and_duplicate_rows", dup, degenerate=True))
    # non-finite rho in one training row: every E-step row falls back to uniform gamma, pi stays 1/S
    r, p = plda(base, 32)
    r[5, 3] = np.nan
    cases += [make("rho_nan", base, rho=r), make("rho_nan_chunks", base, rho=r, chunk=chunks_of(300))]
    # (init_smoothing 0 below does the same from the start: S bit-identical centroids, every score tied, label 0)
    cases.append(make("nan_emb_chunks", _with(base, [2, 3, 150], np.nan), chunk=chunks_of(300, 3)))
    # AHC refuses D >= 7 197: identity labels, S = Tn
    cases.append(make("wide_7197", blobs(40, D_REFUSED, 3, 3), R=16, degenerate=True, ahc="refused",
                      oracle_initial="identity"))
    # shapes: N on the 128-row block edges, emb_dim on the block edges, rho_dim beyond emb_dim
    for n in (1, 2, 3, 127, 128, 129, 255, 256, 257):
        cases.append(make(f"n{n}", blobs(n, 64, min(3, n), 10 + n)))
    for d in (1, 2, 127, 128, 129, 2048):
        cases.append(make(f"emb{d}", blobs(200, d, 3, 20 + d), degenerate=d == 1))
    for R in (1, 2, 33, 300):
        cases.append(make(f"rho{R}", blobs(200, 64, 3, 30 + R), R=R, psi=R != 33, degenerate=R == 1))
    # config edges
    mid = blobs(150, 64, 4, 4)
    cases += [make("threshold_0", mid, cfg=config(threshold=0.0), degenerate=True),
              make("threshold_2.5", mid, cfg=config(threshold=2.5))]
    cases += [make(f"max_it_{m}", mid, cfg=config(max_iterations=m)) for m in (0, 1, 2)]
    cases += [make(f"epsilon_{e}", mid, cfg=config(epsilon=e)) for e in (0.0, 1e300)]
    cases += [make(f"smoothing_{s}", mid, cfg=config(init_smoothing=s)) for s in (0.0, 1.0, 30.0)]
    cases += [make(f"Fa_{f}", mid, cfg=config(Fa=f)) for f in (0.01, 5.0)]
    cases += [make(f"Fb_{f}", mid, cfg=config(Fb=f)) for f in (0.01, 5.0)]
    cases.append(make("min_speakers_1", mid, cfg=config(min_speakers=1)))
    cases.append(make("num_speakers_1_chunks", mid, cfg=config(num_speakers=1), chunk=chunks_of(150), adjusted=True))
    # constrained assignment: one cluster (plain argmax), a chunk with more local speakers than clusters (-2)
    cases.append(make("k1_chunks", blobs(120, 64, 1, 6), chunk=chunks_of(120, 3)))
    ch = chunks_of(300, 2)
    ch[:12] = 0
    cases.append(make("chunk_overflow", base, chunk=np.ascontiguousarray(ch)))
    return {c["name"]: c for c in cases}


CASES = build_cases()


@pytest.mark.parametrize("name", list(CASES))
def test_case_against_oracle_and_standalone_calls(gpu_lib, oracle, name):
    case = CASES[name]
    run = pipeline(case)
    assert run["status"] == 0, (name, run["error"])
    comp = compose(case)
    check_composition(case, run, comp)
    check_oracle(oracle, case, run)
    # the branch the case was built for, confirmed by the info and the launch count
    info, N = run["info"], case["emb"].shape[0]
    assert bool(info["was_adjusted"]) == case["adjusted"], name
    if case["ahc"] in ("refused", "nan"):
        assert info["initial_clusters"] == info["training_count"], name
    want = pipeline_launches(N, info, case["rho"].shape[1], case["cfg"].vbx.max_iterations, ahc=case["ahc"],
                             kmeans=comp["kmeans"])
    assert run["launches"] == want, (name, run["launches"], want)
    labels = run["labels"]
    if name == "chunk_overflow":
        assert (labels == -2).any() and (labels[12:] >= 0).all()
    elif case["chunk"] is not None:
        assert (labels >= 0).all(), name
    if name in ("rho_nan", "smoothing_0.0"):   # uniform gamma everywhere: S equal centroids, the first one wins
        assert info["centroid_count"] == info["initial_clusters"] and (labels == 0).all(), name
    if name == "one_finite":
        assert info["training_count"] == 1 and info["initial_clusters"] == 1
    if name == "two_finite":
        assert info["training_count"] == 2
    if name == "all_nonfinite":
        assert info["training_count"] == N and (labels == 0).all()


# ---- outputs ------------------------------------------------------------------------------------------------------
def test_null_outputs_give_the_same_labels(gpu_lib):
    for name in ("nan_emb_chunks", "rho_nan", "plain"):
        case = CASES[name]
        full = pipeline(case)
        assert full["status"] == 0
        for mask in range(8):
            wi, wc, wf = bool(mask & 1), bool(mask & 2), bool(mask & 4)
            r = pipeline(case, want_initial=wi, want_centroids=wc, want_info=wf)
            assert r["status"] == 0 and np.array_equal(r["labels"], full["labels"]), (name, mask)
            if wi:
                assert np.array_equal(r["initial"], full["initial"])
            if wc:
                assert r["centroids"].tobytes() == full["centroids"].tobytes()
            if wf:
                assert r["info"] == full["info"]


def test_max_centroids_writes_only_the_first_rows(gpu_lib):
    for name in ("plain", "threshold_0"):
        case = CASES[name]
        full = pipeline(case)
        K, E = full["info"]["centroid_count"], case["emb"].shape[1]
        assert K >= 2
        for mc in (0, 1, K - 1, K, K + 3):
            r = pipeline(case, max_centroids=mc)
            assert r["status"] == 0 and np.array_equal(r["labels"], full["labels"])
            kc = min(K, mc)
            assert r["centroids"][:kc].tobytes() == full["centroids"][:kc].tobytes(), (name, mc)
            assert (r["centroids"][kc:] == SENTINEL).all(), (name, mc)
            assert r["centroids"].shape == (max(mc, 1), E)


# ---- the merge kernel's capacity, and the runtime's last error --------------------------------------------------
def test_past_the_merge_capacity_fails_and_leaves_the_thread_clean(gpu_lib):
    """N = W * 2 048 + 1 at D = 4: AHC refuses it, the pipeline falls back to identity labels (S = N), and VBx then asks
    for N^2 doubles, which the device refuses at once.  The next call on the same thread, of the pipeline or of
    another entry point, must not see that stale error."""
    import torch
    from fluidaudio_b200.mel import AudioMelSpectrogram
    L = _lib.load()
    W = torch.cuda.get_device_properties(0).multi_processor_count - 1
    n = W * 2048 + 1
    rng = np.random.default_rng(8)
    big = dict(name="capacity+1", emb=rng.standard_normal((n, 4)).astype(np.float32), rho=rng.standard_normal((n, 4)),
               psi=None, cfg=config(), chunk=None)
    small = CASES["nan_emb_chunks"]
    first = pipeline(small)
    assert first["status"] == 0
    x = rng.standard_normal((50, 16))
    norm0 = np.zeros_like(x)
    _ok(L.fa_l2_normalize_rows(x.ctypes.data, 50, 16, norm0.ctypes.data), "normalize")
    mel = AudioMelSpectrogram(n_mels=80)
    audio = synth.tone_noise_audio(16000)
    mel0 = mel.compute_flat_transposed(audio)[0].copy()

    def fail():
        r = pipeline(big, want_initial=False, want_centroids=False)
        assert r["status"] == 4, (r["status"], r["error"])             # FA_ALLOCATION_FAILURE
        assert "cudaMalloc(" in r["error"] and "out of memory" in r["error"], r["error"]
        assert r["launches"] == 3, r["launches"]                      # widen, finite rows, normalise; no AHC launch
    fail()
    again = pipeline(small)
    assert again["status"] == 0, again["error"]
    for k in ("labels", "initial", "centroids"):
        assert again[k].tobytes() == first[k].tobytes(), k
    assert again["info"] == first["info"]
    fail()
    norm1 = np.zeros_like(x)
    assert L.fa_l2_normalize_rows(x.ctypes.data, 50, 16, norm1.ctypes.data) == 0, L.fa_last_error()
    assert norm1.tobytes() == norm0.tobytes()
    fail()
    assert mel.compute_flat_transposed(audio)[0].tobytes() == mel0.tobytes()
    mel.close()


# ---- history independence -----------------------------------------------------------------------------------------
HISTORY = ["emb2048", "n1", "threshold_0", "one_finite", "rho300", "all_nonfinite", "nan_first_row", "n2", "rho_nan",
           "wide_7197", "k1_chunks", "chunk_overflow"]


def _bytes(r):
    return (r["status"], r["labels"].tobytes(), r["initial"].tobytes(), r["centroids"].tobytes(), tuple(r["info"].items()))


def test_results_do_not_depend_on_earlier_calls(gpu_lib):
    """Contexts are pooled and every arena only grows: a call sees what the previous one left.  Two orders of the same
    mix of sizes and branches (large, small, large) must give the same bytes."""
    a = {n: _bytes(pipeline(CASES[n])) for n in HISTORY}
    order = HISTORY[::2][::-1] + HISTORY[1::2]
    b = {n: _bytes(pipeline(CASES[n])) for n in order}
    for n in HISTORY:
        assert a[n] == b[n], n


def test_concurrent_pipelines_equal_their_sequential_runs(gpu_lib):
    names = ["plain", "nan_emb_chunks", "rho_nan", "threshold_0", "n129", "emb129", "rho_nan_chunks", "two_finite"]
    want = {n: _bytes(pipeline(CASES[n])) for n in names}
    got, errors = {n: [] for n in names}, []

    def worker(n):
        try:
            for _ in range(3):
                got[n].append(_bytes(pipeline(CASES[n])))
        except Exception as ex:   # reported below: an exception in a thread does not fail the test by itself
            errors.append((n, repr(ex)))
    threads = [threading.Thread(target=worker, args=(n,)) for n in names]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for n in names:
        assert len(got[n]) == 3 and all(g == want[n] for g in got[n]), n


# ---- batch --------------------------------------------------------------------------------------------------------
BATCH_MIX = ["plain", "nan_first_row", "rho_nan", "one_finite", "all_nonfinite", "n1", "n2", "nan_last_element",
             "inf_rows", "two_finite", "n3", "n127"]


def batch(sets, with_chunks, lead=3, tail=5, empty_at=(), offsets=None):
    """One fa_diarize_cluster_batch(_chunks) call over `sets` (case names), with `lead` / `tail` rows outside every set
    and empty sets inserted before the positions in `empty_at`.  All sets share E = 64 and R = 32."""
    L = _lib.load()
    embs, rhos, chunks, offs, names = [], [], [], [lead], []
    for i, n in enumerate(sets):
        for _ in range(empty_at.count(i)):
            offs.append(offs[-1])
            names.append(None)
        c = CASES[n]
        embs.append(c["emb"])
        rhos.append(c["rho"])
        chunks.append(c["chunk"] if c["chunk"] is not None else chunks_of(c["emb"].shape[0]))
        offs.append(offs[-1] + c["emb"].shape[0])
        names.append(n)
    for _ in range(empty_at.count(len(sets))):
        offs.append(offs[-1])
        names.append(None)
    rng = np.random.default_rng(len(sets))
    total = offs[-1] + tail
    emb = np.concatenate([rng.standard_normal((lead, 64)).astype(np.float32)] + embs +
                         [rng.standard_normal((tail, 64)).astype(np.float32)])
    rho = np.concatenate([np.zeros((lead, 32))] + rhos + [np.zeros((tail, 32))])
    chunk = np.concatenate([np.zeros(lead, np.int32)] + chunks + [np.zeros(tail, np.int32)])
    off = np.array(offs if offsets is None else offsets, np.int64)
    count = off.size - 1
    labels = np.full(total, -9, np.int32)
    infos = (_lib.ClusterInfo * max(count, 1))()
    for i in range(count):   # pre-filled: an empty set's info must be zeroed
        infos[i].training_count = 77
    psi = CASES["plain"]["psi"]
    cfg = config()
    before = L.fa_kernel_launch_count()
    if with_chunks:
        st = L.fa_diarize_cluster_batch_chunks(emb.ctypes.data, rho.ctypes.data, off.ctypes.data, count, 64, 32,
                                               psi.ctypes.data, C.byref(cfg), chunk.ctypes.data, labels.ctypes.data,
                                               infos)
    else:
        st = L.fa_diarize_cluster_batch(emb.ctypes.data, rho.ctypes.data, off.ctypes.data, count, 64, 32,
                                        psi.ctypes.data, C.byref(cfg), labels.ctypes.data, infos)
    return dict(status=int(st), labels=labels, infos=[info_dict(infos[i]) for i in range(count)], offsets=off,
                names=names, launches=L.fa_kernel_launch_count() - before, lead=lead, tail=tail)


def _single(name, with_chunks):
    c = dict(CASES[name])
    c["cfg"] = config()
    c["psi"] = CASES["plain"]["psi"]
    if with_chunks:
        c["chunk"] = c["chunk"] if c["chunk"] is not None else chunks_of(c["emb"].shape[0])
    else:
        c["chunk"] = None
    return pipeline(c)


@pytest.mark.parametrize("with_chunks", [False, True])
@pytest.mark.parametrize("count", [1, 2, 5, 9, 33])
def test_batch_equals_single_calls(gpu_lib, count, with_chunks):
    sets = [BATCH_MIX[i % len(BATCH_MIX)] for i in range(count)]
    empty_at = (0, count // 2, count) if count >= 2 else (count,)
    b = batch(sets, with_chunks, empty_at=empty_at)
    assert b["status"] == 0, _lib.load().fa_last_error()
    assert (b["labels"][:b["lead"]] == -9).all() and (b["labels"][b["labels"].size - b["tail"]:] == -9).all()
    singles = {n: _single(n, with_chunks) for n in set(sets)}
    off = b["offsets"]
    for m, n in enumerate(b["names"]):
        if n is None:
            assert off[m + 1] == off[m] and b["infos"][m] == dict.fromkeys(INFO_FIELDS, 0), m
            continue
        s = singles[n]
        assert np.array_equal(b["labels"][off[m]:off[m + 1]], s["labels"]), (m, n)
        assert b["infos"][m] == s["info"], (m, n, b["infos"][m], s["info"])
    again = batch(sets, with_chunks, empty_at=empty_at)
    assert again["status"] == 0 and again["labels"].tobytes() == b["labels"].tobytes() and again["infos"] == b["infos"]


def test_batch_rejects_bad_offsets_before_any_launch(gpu_lib):
    sets = ["plain", "n3", "n127"]
    for bad in ([3, 303, 300, 430], [-1, 303, 306, 433], [3, 306, 303, 433]):
        b = batch(sets, False, offsets=bad)
        assert b["status"] == 1, bad                                   # FA_INVALID_ARGUMENT
        assert b["launches"] == 0 and (b["labels"] == -9).all(), bad
        assert "set_offsets" in _lib.load().fa_last_error().decode()


def test_report():
    print(f"\npipeline sweep: {len(CASES)} cases, worst centroid deviation {WORST[0]:.2e} x 1e-9, "
          f"{time.perf_counter() - T_START:.1f} s")
