"""Sortformer streaming state on the H100 against the oracle across its configuration space, bit for bit after every
push (the confirmed and tentative rows, the model inputs and the pushed sessions' full snapshots):

* all eight presets at 1, 7 and 64 sessions, every stream through at least three compressions, the adversarial
  generators of ``sortformer_cases`` mixed in with synth.sortformer_chunk's;
* every edge configuration of ``sortformer_cases.EDGE_CONFIGS`` at 7 sessions, which must also reach the branch it is
  listed for;
* one push of 4 096 sessions in which every session compresses in the same launch;
* three handles with different configurations and shared-memory needs alive at once, their pushes interleaved;
* the largest max_core_frames whose compression fits the kernel's shared memory, and one frame more refused at create.

Host and device variants alternate.  Each test prints what it covered: compressions, ties decided by index in each
selection, kept -inf (maxIndex) slots and disabled slots filled with the silence mean.  NaN predictions are out of
scope: vDSP.clip leaves their meaning undefined.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

import sortformer_cases as cases
from fluidaudio_b200 import _lib
from fluidaudio_b200.sortformer import PRESETS, SortformerConfig, SortformerStreams
from sortformer_cases import Harness, same_state

D, S = 512, 4
MODES = cases.ALL_MODES + ("offline",)
SMEM_LIMIT = 200 * 1024   # sortformer_kernels.cu: the update kernel's dynamic shared-memory ceiling


@pytest.fixture(scope="module")
def O():
    from oracle import oracle_sortformer
    oracle_sortformer.build()
    oracle_sortformer.lib()
    return oracle_sortformer


def run_until(H, need, streaming_every=3, max_steps=4000):
    """push varying subsets of the live sessions in varying orders until each has had ``need`` compressions"""
    step = 0
    while min(H.compressions[s] for s in H.ref) < need:
        assert step < max_steps, dict(H.compressions)
        streaming_rule = step % streaming_every == 0
        live = [s for s in H.ref if H.compressions[s] < need] or list(H.ref)
        k = max(1, int(len(live) * H.rng.uniform(0.5, 1.0)))
        H.push([int(s) for s in H.rng.permutation(live)[:k]], device=step % 2 == 1, streaming_rule=streaming_rule)
        step += 1
    for sid in H.ref:
        same_state(H.h.state(sid), H.ref[sid].state())


@pytest.mark.gpu
@pytest.mark.parametrize("preset", PRESETS)
@pytest.mark.parametrize("sessions", [1, 7, 64])
def test_presets_match_the_oracle(gpu_lib, O, preset, sessions):
    H = Harness(O, SortformerConfig.preset(preset), seed=sessions * 7919 + PRESETS.index(preset))
    for i in range(sessions):
        H.open(MODES[(i + PRESETS.index(preset)) % len(MODES)])
    run_until(H, 3)
    print(H.cov.line(f"{preset} x {sessions}"))
    assert H.cov.c["compressions"] >= 3 * sessions


@pytest.mark.gpu
@pytest.mark.parametrize("edge", cases.EDGE_CONFIGS, ids=cases.EDGE_IDS)
def test_edge_configs_match_the_oracle(gpu_lib, O, edge):
    cfg, resolved, max_core = cases.edge_config(edge)
    H = Harness(O, cfg, seed=zlib.crc32(edge.name.encode()), max_core=max_core)
    assert (H.h.config, H.h.max_core) == (resolved, max_core)
    H.long_chunks = True   # contexts as sortformer_cases.contexts draws them: short or long chunks for offline edges
    for i in range(7):
        H.open(edge.modes[i % len(edge.modes)])
    run_until(H, 3, streaming_every=1 if not edge.offline else 3)
    print(H.cov.line(edge.name))
    assert edge.reached(H.cov), (edge.reaches, dict(H.cov.c), sorted(H.cov.sizes))


@pytest.mark.gpu
def test_4096_sessions_compress_in_one_launch(gpu_lib, O):
    """every push after the second compresses every session: 4 096 compressions in one launch, three times"""
    cfg = SortformerConfig(chunk_len=12, chunk_left_context=1, chunk_right_context=3, fifo_len=8, spkcache_len=32,
                           spkcache_update_period=12, spkcache_sil_frames_per_spk=2)
    H = Harness(O, cfg, seed=4096)
    ids = [H.open(MODES[i % len(MODES)]) for i in range(4096)]
    for step in range(5):
        before = H.cov.c["compressions"]
        launches = _lib.kernel_launch_count()
        H.push(ids, device=step % 2 == 1, streaming_rule=True)
        assert H.cov.c["compressions"] - before == (4096 if step >= 2 else 0)
        assert _lib.kernel_launch_count() - launches == 2   # one update, one model-input gather
    print(H.cov.line("4096 sessions"))


@pytest.mark.gpu
def test_three_handles_interleaved(gpu_lib, O):
    """three handles of different configurations (and shared-memory needs) alive at once, pushes interleaved, each
    session checked against its own oracle session"""
    fifo0 = next(e for e in cases.EDGE_CONFIGS if e.name == "fifo0")
    handles = [Harness(O, SortformerConfig.preset("default"), seed=31),
               Harness(O, SortformerConfig(**fifo0.fields), seed=32),
               Harness(O, SortformerConfig(chunk_len=2000), seed=33)]   # about 109 KB of shared memory
    for j, H in enumerate(handles):
        for i in range(3):
            H.open(MODES[(3 * j + i) % len(MODES)])
    step = 0
    while any(min(H.compressions[s] for s in H.ref) < 3 for H in handles):
        assert step < 400
        for j, H in enumerate(handles):
            if min(H.compressions[s] for s in H.ref) < 3:
                H.push(list(H.ref), device=(step + j) % 2 == 1, streaming_rule=True)
        step += 1
    for j, H in enumerate(handles):
        for sid in H.ref:
            same_state(H.h.state(sid), H.ref[sid].state())
        print(H.cov.line(f"handle {j}"))


def update_smem_bytes(spkcache_len, fifo_len, max_core, sil):
    """the compression's shared memory (sortformer_kernels.cu smem_layout): scores [rows x 4], the permuted values and
    their flags [(rows + sil) x 4] each, the slots [spkcacheLen] and the scan [257], each part rounded to 16 bytes"""
    a16 = lambda b: (b + 15) // 16 * 16
    rows = spkcache_len + fifo_len + max_core
    n = (rows + sil) * S
    return a16(rows * S * 4) + 2 * a16(n * 4) + a16(spkcache_len * 4) + a16(257 * 4)


@pytest.mark.gpu
def test_largest_max_core_fits_and_one_more_is_refused(gpu_lib, O):
    cfg = SortformerConfig.preset("default")
    size = lambda m: update_smem_bytes(cfg.spkcache_len, cfg.fifo_len, m, cfg.spkcache_sil_frames_per_spk)
    largest = max(m for m in range(1, 20000) if size(m) <= SMEM_LIMIT)
    assert largest == 3999   # 48 bytes per cache row: (188 + 40 + 3999) * 48 + 1 888 = 204 784
    # one frame more: refused at create, no handle, no launch
    before = _lib.kernel_launch_count()
    h = C.c_void_p()
    assert gpu_lib.fa_sortformer_create(C.byref(cfg.to_c()), largest + 1, C.byref(h)) == 1
    assert h.value is None and _lib.kernel_launch_count() == before
    with pytest.raises(_lib.FluidAudioError):
        SortformerStreams(cfg, largest + 1)
    # the largest: accepted, and two pushes of that many core frames compress as the oracle does
    H = Harness(O, cfg, seed=3999, max_core=largest)
    sids = [H.open("turns"), H.open("quantized")]
    H.contexts = lambda sid, rule: (largest, cfg.chunk_left_context if H.ref[sid].chunks else 0,
                                    cfg.chunk_right_context)
    for step in range(2):
        H.push(sids, device=step == 1, streaming_rule=False)
    assert H.cov.c["compressions"] == 4 and max(H.cov.sizes) > 4 * 4000
    print(H.cov.line(f"max_core {largest}"))
