"""Sortformer streaming state on the H100 against the oracle (``oracle/oracle_sortformer.cpp``), bit for bit.

Sessions of four presets (1, 7 and 64 at a time) run seeded streams long enough for at least three compressions each:
turn-taking predictions, predictions on a 1/8 grid (exact ties, exact 0.25 / 0.5 / 0.75), all-silence and never-silent
streams, and offline-style contexts with a short last chunk; every model output is drawn afresh, so the fifoPreds
refresh and the first spkcachePreds take the model's new rows.  Pushes name varying subsets in varying orders, sessions
are closed and their ids reused, and the host and device variants alternate.  After every push the confirmed and
tentative rows, the model inputs and the pushed sessions' full snapshots equal the oracle's.  Also: the launch count of
a push, and that every invalid argument leaves all snapshots unchanged.
"""
import numpy as np
import pytest

from fluidaudio_b200 import _lib, synth
from fluidaudio_b200.sortformer import SortformerConfig, SortformerStreams
from sortformer_cases import Harness, chunks_needed, same_state

D, S = 512, 4
MODES = synth.SORTFORMER_MODES + ("offline",)


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_sortformer
    oracle_sortformer.build()
    oracle_sortformer.lib()
    return oracle_sortformer


@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["default", "balancedV2", "highContextV2", "efficientV2_1"])
@pytest.mark.parametrize("sessions", [1, 7, 64])
def test_streams_match_the_oracle(gpu_lib, O, preset, sessions):
    cfg = SortformerConfig.preset(preset)
    H = Harness(O, cfg, seed=sessions * 1000 + len(preset))
    for i in range(sessions):
        H.open(MODES[i % len(MODES)])
    need = chunks_needed(H.h.config)
    reopened, step = 0, 0
    while min(r.chunks for r in H.ref.values()) < need:
        live = list(H.ref)
        streaming_rule = step % 3 == 0
        pool = [s for s in live if not (streaming_rule and H.mode[s] == "offline")] or live[:0]
        if not pool:
            step += 1
            continue
        k = max(1, int(len(pool) * H.rng.uniform(0.5, 1.0)))
        ids = [int(s) for s in H.rng.permutation(pool)[:k]]
        H.push(ids, device=step % 2 == 1, streaming_rule=streaming_rule)
        # now and then a finished session closes and a new one reuses the lowest free id
        if sessions > 1 and step % 17 == 16 and reopened < 3:
            sid = max(H.ref, key=lambda s: H.ref[s].chunks)
            if H.ref[sid].chunks >= need:
                mode = H.mode[sid]
                reopened += 1
                H.close(sid)
                assert H.open(mode) == sid   # the lowest free id
        step += 1
    for sid in H.ref:
        same_state(H.h.state(sid), H.ref[sid].state())
    comps = [1 for r in H.ref.values() if r.lengths().has_spkcache_preds]
    assert len(comps) == len(H.ref)


@pytest.mark.gpu
def test_basic_flow_with_48_core_frames(gpu_lib, O):
    cfg = SortformerConfig.preset("default")
    H = Harness(O, cfg, seed=3, max_core=48)
    sid = H.open("turns")
    rows = 48 + cfg.chunk_left_context + cfg.chunk_right_context
    conf, tent = H.h.update([sid], np.zeros((1, rows, D), np.float32), np.zeros((1, rows, S), np.float32),
                            left_context=[cfg.chunk_left_context], right_context=[cfg.chunk_right_context])
    assert conf[0].size == 48 * 4 and tent[0].size == cfg.chunk_right_context * 4


def _launches(fn):
    before = _lib.kernel_launch_count()
    fn()
    _lib.synchronize()
    return _lib.kernel_launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("sessions", [1, 64])
def test_launch_count_of_a_push(gpu_lib, O, sessions):
    from fluidaudio_b200.sortformer import step_lengths
    cfg = SortformerConfig.preset("default")
    H = Harness(O, cfg, seed=5)
    ids = [H.open("turns") for _ in range(sessions)]
    rng = np.random.default_rng(1)
    rows_max = cfg.chunk_left_context + cfg.chunk_len + cfg.chunk_right_context
    pred_max = cfg.spkcache_len + cfg.fifo_len + rows_max
    dE, dP = _lib.DeviceBuffer(4 * sessions * rows_max * D), _lib.DeviceBuffer(4 * sessions * pred_max * S)
    dc, dt = _lib.DeviceBuffer(4 * sessions * rows_max * S), _lib.DeviceBuffer(4 * sessions * rows_max * S)
    dsc, dff = _lib.DeviceBuffer(4 * sessions * cfg.spkcache_len * D), _lib.DeviceBuffer(4 * sessions * cfg.fifo_len * D)
    compressing = {"host": 0, "device": 0}
    step = 0
    while min(compressing.values()) < 2:   # the first compression comes after (188 + 40 + 31) / 6 chunks
        assert step < 200
        variant = "device" if step % 2 else "host"
        rows = cfg.chunk_len + cfg.chunk_right_context + (cfg.chunk_left_context if step else 0)
        st = H.h.state(ids[0])   # every session has the same lengths
        plan = step_lengths(cfg, st.spkcache_length, st.fifo_length, st.has_spkcache_preds, rows, pred_max,
                            cfg.chunk_left_context if step else 0, cfg.chunk_right_context)
        E = rng.normal(size=(sessions, rows, D)).astype(np.float32)
        P = rng.uniform(size=(sessions, pred_max, S)).astype(np.float32)
        if variant == "host":
            assert _launches(lambda: H.h.update(ids, E, P)) == 1            # one update kernel
            assert _launches(lambda: H.h.model_inputs(ids)) == 1           # one gather kernel
        else:
            dE.upload(E)
            dP.upload(P)
            assert _launches(lambda: H.h.update_device(ids, dE, rows, dP, pred_max, dc, dt)) == 1
            assert _launches(lambda: H.h.model_inputs_device(ids, dsc, dff)) == 1
        compressing[variant] += plan.compress
        step += 1
    assert H.h.state(ids[-1]).has_spkcache_preds
    assert _launches(lambda: H.h.update([], np.zeros((0, 1, D), np.float32), np.zeros((0, 1, S), np.float32))) == 0
    for b in (dE, dP, dc, dt, dsc, dff):
        b.free()


@pytest.mark.gpu
def test_handles_of_different_shared_memory_sizes(gpu_lib, O):
    """A handle whose compression needs more than the default 48 KB of shared memory keeps working after a smaller
    handle is created: the kernel's shared-memory ceiling is not per handle."""
    big = Harness(O, SortformerConfig(chunk_len=2000), seed=11)   # 2 228 cache rows before compression: about 109 KB
    small = Harness(O, SortformerConfig.preset("default"), seed=12)
    assert big.h.config.spkcache_update_period == 2000 and big.h.max_core == 2000
    b, s = big.open("turns"), small.open("turns")
    for step in range(3):
        big.push([b], device=step % 2 == 1, streaming_rule=True)   # every push pops 2 000 rows and compresses
        assert big.ref[b].last_compression() is not None
        small.push([s], device=step % 2 == 0, streaming_rule=True)


@pytest.mark.gpu
def test_model_inputs_of_more_sessions_than_a_grid_row(gpu_lib):
    """The model-input gather puts sessions on grid x: 70 000 sessions in one call (grid y would stop at 65 535)."""
    cfg = SortformerConfig(chunk_len=1, chunk_left_context=0, chunk_right_context=0, fifo_len=0, spkcache_len=16,
                           spkcache_update_period=1)
    sf = SortformerStreams(cfg)
    n = 70000
    ids = np.array([sf.open() for _ in range(n)], np.int32)
    E = np.arange(n, dtype=np.float32)[:, None, None] + np.zeros((1, 1, D), np.float32)   # session i's row: all i
    P = np.full((n, 1, S), 0.5, np.float32)
    sf.update(ids, E, P)   # fifoLen 0: the row is popped straight into the speaker cache
    dsc, dff = _lib.DeviceBuffer(4 * n * cfg.spkcache_len * D), _lib.DeviceBuffer(4)
    sl, fl = sf.model_inputs_device(ids, dsc, dff)
    _lib.synchronize()
    assert (sl == 1).all() and (fl == 0).all()
    for i in (0, 65534, 65535, 65536, n - 1):
        got = np.empty((cfg.spkcache_len, D), np.float32)
        _lib.check(gpu_lib.fa_memcpy_d2h(got.ctypes.data, dsc.ptr.value + 4 * i * cfg.spkcache_len * D, got.nbytes),
                   "fa_memcpy_d2h")
        assert (got[0] == i).all() and not got[1:].any(), i
    dsc.free()
    dff.free()
    sf.close_handle()


@pytest.mark.gpu
def test_invalid_arguments_leave_every_session_unchanged(gpu_lib, O):
    cfg = SortformerConfig.preset("default")
    H = Harness(O, cfg, seed=9)
    ids = [H.open(m) for m in ("turns", "quantized", "silence")]
    closed = H.open("turns")
    H.close(closed)
    for step in range(40):
        H.push(ids, device=step % 2 == 1, streaming_rule=True)
    before = [H.h.state(s) for s in ids]
    L = gpu_lib
    c = H.h.config
    lc, rc, core = c.chunk_left_context, c.chunk_right_context, c.chunk_len
    n = [H.ref[s].lengths() for s in ids]
    er = lc + core + rc
    pr = max(x.spkcache_length + x.fifo_length for x in n) + er
    E, P = np.zeros((3, er, D), np.float32), np.full((3, pr, S), 0.3, np.float32)

    def call(sessions, E=E, P=P, el=None, lcs=None, rcs=None, conf_len=None, count=None):
        sid = np.array(sessions, np.int32)
        m = sid.size if count is None else count
        el = np.full(m, E.shape[1], np.int32) if el is None else np.array(el, np.int32)
        out = np.zeros(max(1, m * E.shape[1] * S), np.float32)
        cr, tr = np.zeros(max(m, 1), np.int64), np.zeros(max(m, 1), np.int64)
        return L.fa_sortformer_update(H.h._h, m, sid.ctypes.data, E.ctypes.data, E.shape[1], P.ctypes.data, P.shape[1],
                                      el.ctypes.data, _lib.ptr(lcs), _lib.ptr(rcs), out.ctypes.data,
                                      out.size if conf_len is None else conf_len, out.ctypes.data, out.size,
                                      cr.ctypes.data, tr.ctypes.data)

    cases = {
        "duplicate": call([ids[0], ids[1], ids[0]]),
        "closed": call([ids[0], closed, ids[1]], count=3),
        "insufficient preds": call(ids, P=np.ascontiguousarray(P[:, :er])),
        "core above max_core": call(ids, E=np.zeros((3, er + 1, D), np.float32)),
        "negative core": call(ids, el=[er, 2, er]),
        "negative context": call(ids, lcs=np.array([1, -1, 1], np.int32), rcs=np.array([rc] * 3, np.int32)),
        "confirmed too small": call(ids, conf_len=core * S * 3 - 1),
        "emb length above rows": call(ids, el=[er, er + 1, er]),
    }
    assert all(v == 1 for v in cases.values()), cases
    for s, b in zip(ids, before):
        same_state(H.h.state(s), b)
    H.push(ids, device=False, streaming_rule=True)   # and the sessions go on as the oracle does
