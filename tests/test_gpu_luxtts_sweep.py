"""LuxTTS synthesis on the H100 against the oracle (oracle/oracle_luxtts.cpp): begin's RMS, noise, conditions and
reasons; text conditions at several row strides; interleaved steps; the vocoder input at both buckets; finish with
non-finite and out-of-range samples and the capacity refusal; host and device variants with their launch counts; the
end-to-end pipeline with deterministic fake models; and the reference's own fixture prompt."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200 import luxtts as LX
from fluidaudio_b200.mel import LuxTtsMelExtractor
from oracle import oracle_luxtts as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "luxtts")
MASK = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module", autouse=True)
def device():
    if _lib.device_count() < 1:
        pytest.skip("needs an H100")
    _lib.set_device(0)


@pytest.fixture(scope="module")
def mel():
    return LuxTtsMelExtractor()


def _uniform(s0, k):
    z = (s0 + k * GAMMA) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    z ^= z >> 31
    u = float(z >> 11) / float(1 << 53)
    return u if u > 0 else 2.2250738585072014e-308


def _noise_exceptions(got, want, seed):
    """indices where got != want; each must be the float32 neighbour of a float64 value within 2^-40 of a midpoint"""
    s0 = 0xdeadbeefcafebabe if seed == 0 else seed
    bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
    for j in bad.tolist():
        d = math.sqrt(-2.0 * math.log(_uniform(s0, 2 * j + 1))) * math.cos(2.0 * math.pi * _uniform(s0, 2 * j + 2))
        a, b = float(got[j]), float(want[j])
        assert abs(int(got[j:j + 1].view(np.int32)[0]) - int(want[j:j + 1].view(np.int32)[0])) == 1, j
        assert abs(d - (a + b) / 2) <= 2.0 ** -40 * abs(d), (j, d, a, b)
    return bad.size


def _prompts(rng, n, seconds=(0.3, 5.5)):
    out = []
    for i in range(n):
        m = int(rng.integers(int(seconds[0] * 24000), int(seconds[1] * 24000)))
        scale = (0.01, 0.05, 0.3)[i % 3]
        out.append((rng.normal(size=m) * scale).astype(np.float32))
    return out


def _begin_case(rng, n):
    prompts = _prompts(rng, n)
    pt = rng.integers(20, 80, size=n).astype(np.int32)
    tt = rng.integers(10, 100, size=n).astype(np.int32)
    speeds = rng.choice(np.array([0.8, 1.0, 1.3], np.float32), size=n)
    seeds = rng.integers(0, 2**63, size=n).astype(np.uint64)
    seeds[0] = 0
    ok = np.array([O.plan(p.size, a, b, s)[0] == 0 for p, a, b, s in zip(prompts, pt, tt, speeds)])
    keep = np.flatnonzero(ok)
    return [prompts[i] for i in keep], pt[keep], tt[keep], speeds[keep], seeds[keep]


# ------------------------------------------------------------------------------------------------ begin
@pytest.mark.parametrize("n", [1, 7, 64, 1024])
def test_begin_equals_the_oracle(mel, n):
    rng = np.random.default_rng(n)
    prompts, pt, tt, speeds, seeds = _begin_case(rng, n)
    R = LX.LuxTtsRequests()
    ids, plans, sc, pm = R.begin(prompts, pt, tt, speeds, seeds)
    exceptions = 0
    check = range(len(ids)) if len(ids) <= 64 else rng.choice(len(ids), 48, replace=False)
    for i in check:
        p, plan = prompts[i], plans[i]
        r, ns, P, S, L, G, B = O.plan(p.size, pt[i], tt[i], speeds[i])
        assert (plan.reason, plan.prompt_samples, plan.prompt_frames, plan.token_count, plan.features_length,
                plan.gen_frames, plan.bucket) == (r, ns, P, S, L, G, B)
        rms = O.rms(p[:ns])
        assert np.float32(plan.prompt_rms).tobytes() == rms.tobytes()
        assert plan.boosted == (rms < np.float32(0.1))
        gained = O.gain(p[:ns], rms)
        m = mel.extract(gained)
        want = np.zeros((1024, 100), np.float32)
        want[:P] = (m * np.float32(0.1)).astype(np.float32)
        assert sc[i].tobytes() == want.tobytes()
        assert pm[i].tobytes() == np.where(np.arange(1024) >= L, 1, 0).astype(np.float32).tobytes()
        _, x = R.state(int(ids[i]))
        wx = np.zeros(102400, np.float32)
        wx[:L * 100] = O.noise(int(seeds[i]), L * 100)
        assert x.reshape(-1)[L * 100:].tobytes() == wx[L * 100:].tobytes()
        exceptions += _noise_exceptions(x.reshape(-1)[:L * 100], wx[:L * 100], int(seeds[i]))
    print(f"noise exceptions: {exceptions} over {len(check)} requests")
    R.close_handle()


def test_begin_reasons_and_refusal_change_nothing():
    rng = np.random.default_rng(3)
    R = LX.LuxTtsRequests()
    good = (rng.normal(size=30000) * 0.2).astype(np.float32)
    ids, _, _, _ = R.begin([good], [30], [40], [1.0], [1])
    cases = [(good, 0, 5, 1.0), (good, 5, 0, 1.0), (np.zeros(0, np.float32), 5, 5, 1.0), (good, 5, 5, float("nan")),
             (np.zeros(5000, np.float32), 5, 5, 1.0), (good[:100], 5, 5, 1.0), (good, 200, 60, 1.0),
             (good, 5, 200, 1.0), (good, 60, 1, 100.0), (good, 10, 100, 0.5), (good[:512], 150, 5, 1.0)]
    for audio, a, b, s in cases:
        want = O.plan(audio.size, a, b, s)[0] if audio.any() or audio.size == 0 else 5
        with pytest.raises(LX.LuxTtsError) as e:
            R.begin([good, audio], [30, a], [40, b], [1.0, s], [2, 3])
        assert e.value.reasons.tolist() == [0, want]
    with pytest.raises(_lib.FluidAudioError):
        R.state(1)   # nothing was opened: id 1 is still closed
    nid, _, _, _ = R.begin([good], [30], [40], [1.0], [1])
    assert nid.tolist() == [1]
    R.close_handle()


# ------------------------------------------------------------------------------------------------ conditions and steps
def test_text_condition_at_row_strides():
    rng = np.random.default_rng(4)
    prompts, pt, tt, speeds, seeds = _begin_case(rng, 12)
    R = LX.LuxTtsRequests()
    ids, plans, _, _ = R.begin(prompts, pt, tt, speeds, seeds)
    for stride in (100, 112, 128):
        emb = rng.normal(size=(len(ids), 256, stride)).astype(np.float32)
        got = R.text_condition(ids, emb)
        for i, p in enumerate(plans):
            want, _, _ = O.conditions(emb[i, :p.token_count + 1, :100], p.token_count, p.features_length,
                                      np.zeros((p.prompt_frames, 100), np.float32))
            assert got[i].tobytes() == want.tobytes()
    R.close_handle()


def test_interleaved_steps_vocoder_and_finish():
    rng = np.random.default_rng(5)
    prompts, pt, tt, speeds, seeds = _begin_case(rng, 40)
    R = LX.LuxTtsRequests()
    ids, plans, _, _ = R.begin(prompts, pt, tt, speeds, seeds)
    xs = {int(r): R.state(int(r))[1].reshape(-1).copy() for r in ids}
    steps = {int(r): 0 for r in ids}
    while any(s < 4 for s in steps.values()):
        live = [r for r in ids if steps[int(r)] < 4]
        sel = rng.choice(live, size=max(1, len(live) // 2), replace=False)
        x, t = R.model_inputs(sel)
        v = rng.normal(size=(len(sel), 1024, 112)).astype(np.float32)
        R.advance(sel, v)
        for j, r in enumerate(sel.tolist()):
            p = plans[list(ids).index(r)]
            assert x[j].reshape(-1).tobytes() == xs[r].tobytes()
            assert t[j] == np.float32(O.time_steps()[steps[r]])
            L = p.features_length
            xs[r][:L * 100] = O.step(xs[r][:L * 100], v[j, :L, :100].reshape(-1), steps[r])
            steps[r] += 1
    for r in ids:
        assert R.state(int(r))[1].reshape(-1).tobytes() == xs[int(r)].tobytes()
    for bucket in (282, 555):
        sel = np.array([r for r, p in zip(ids, plans) if p.bucket == bucket], np.int32)
        if not sel.size:
            continue
        mel = R.vocoder_input(sel, bucket)
        for j, r in enumerate(sel.tolist()):
            p = plans[list(ids).index(r)]
            assert mel[j].tobytes() == O.vocoder_input(xs[r], p.prompt_frames, p.gen_frames, bucket).tobytes()
        rows = 300000
        audio = (rng.normal(size=(sel.size, rows)) * 1.5).astype(np.float32)
        audio[:, 3], audio[:, 7], audio[:, 11] = np.nan, np.inf, -np.inf
        lengths, total = np.zeros(sel.size, np.int64), C.c_int64()
        small = np.empty(10, np.float32)
        st = _lib.load().fa_luxtts_finish(R._h, sel.size, sel.ctypes.data, audio.ctypes.data, rows, rows,
                                          small.ctypes.data, 10, lengths.ctypes.data, C.byref(total))
        assert st == LX.STATUS_OUTPUT_TOO_SMALL and total.value == lengths.sum() > 10
        out = R.finish(sel, audio)
        for j, r in enumerate(sel.tolist()):
            p = plans[list(ids).index(r)]
            want = O.finish(audio[j], p.gen_frames, np.float32(p.prompt_rms))
            # a NaN stays NaN; the device's min / max and multiply give it the canonical payload
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(out[j]), nan) and out[j][~nan].tobytes() == want[~nan].tobytes()
    R.close_handle()


# ------------------------------------------------------------------------------------------------ device variants
def test_device_variants_equal_host_variants_and_count_launches():
    rng = np.random.default_rng(6)
    prompts, pt, tt, speeds, seeds = _begin_case(rng, 9)
    L = _lib.load()
    host, dev = LX.LuxTtsRequests(), LX.LuxTtsRequests()
    hid, hplans, hsc, hpm = host.begin(prompts, pt, tt, speeds, seeds)
    n = len(hid)
    audio = np.concatenate(prompts)
    off = np.concatenate([[0], np.cumsum([p.size for p in prompts])]).astype(np.int64)
    d_a, d_sc, d_pm = _lib.DeviceBuffer(audio.nbytes), _lib.DeviceBuffer(hsc.nbytes), _lib.DeviceBuffer(hpm.nbytes)
    d_a.upload(audio)
    _lib.synchronize()
    reasons, did = np.zeros(n, np.int32), np.zeros(n, np.int32)
    plans = (_lib.LuxTtsPlanInfo * n)()
    sp, sd = np.ascontiguousarray(speeds, np.float32), np.ascontiguousarray(seeds, np.uint64)
    before = L.fa_kernel_launch_count()
    _lib.check(L.fa_luxtts_begin_device(dev._h, n, d_a.ptr, off.ctypes.data, pt.ctypes.data, tt.ctypes.data,
                                        sp.ctypes.data, sd.ctypes.data, reasons.ctypes.data, did.ctypes.data, plans,
                                        d_sc.ptr, d_pm.ptr), "fa_luxtts_begin_device")
    assert L.fa_kernel_launch_count() - before == 4
    _lib.synchronize()
    assert d_sc.download(hsc.shape, np.float32).tobytes() == hsc.tobytes()
    assert d_pm.download(hpm.shape, np.float32).tobytes() == hpm.tobytes()
    emb = rng.normal(size=(n, 256, 112)).astype(np.float32)
    d_e, d_tc = _lib.DeviceBuffer(emb.nbytes), _lib.DeviceBuffer(n * 409600)
    d_e.upload(emb)
    _lib.synchronize()
    before = L.fa_kernel_launch_count()
    _lib.check(L.fa_luxtts_text_condition_device(dev._h, n, did.ctypes.data, d_e.ptr, 112, 256 * 112, d_tc.ptr), "tc")
    assert L.fa_kernel_launch_count() - before == 1
    _lib.synchronize()
    assert d_tc.download((n, 1024, 100), np.float32).tobytes() == host.text_condition(hid, emb).tobytes()
    d_x, d_t, d_v = _lib.DeviceBuffer(n * 409600), _lib.DeviceBuffer(4 * n), _lib.DeviceBuffer(n * 1024 * 100 * 4)
    for k in range(4):
        x, t = host.model_inputs(hid)
        before = L.fa_kernel_launch_count()
        _lib.check(L.fa_luxtts_model_inputs_device(dev._h, n, did.ctypes.data, d_x.ptr, d_t.ptr), "mi")
        assert L.fa_kernel_launch_count() - before == 1
        _lib.synchronize()
        assert d_x.download(x.shape, np.float32).tobytes() == x.tobytes()
        assert d_t.download(t.shape, np.float32).tobytes() == t.tobytes()
        v = rng.normal(size=(n, 1024, 100)).astype(np.float32)
        host.advance(hid, v)
        d_v.upload(v)
        _lib.synchronize()
        before = L.fa_kernel_launch_count()
        _lib.check(L.fa_luxtts_advance_device(dev._h, n, did.ctypes.data, d_v.ptr, 100, 102400), "adv")
        assert L.fa_kernel_launch_count() - before == 1
    _lib.synchronize()
    for bucket in (282, 555):
        sel = [j for j in range(n) if hplans[j].bucket == bucket]
        if not sel:
            continue
        hs, ds = hid[sel].astype(np.int32), did[sel].astype(np.int32)
        m = host.vocoder_input(hs, bucket)
        d_m = _lib.DeviceBuffer(m.nbytes)
        _lib.check(L.fa_luxtts_vocoder_input_device(dev._h, len(sel), ds.ctypes.data, bucket, d_m.ptr), "voc")
        _lib.synchronize()
        assert d_m.download(m.shape, np.float32).tobytes() == m.tobytes()
        a = (rng.normal(size=(len(sel), 290000)) * 1.2).astype(np.float32)
        want = host.finish(hs, a)
        d_in, d_out = _lib.DeviceBuffer(a.nbytes), _lib.DeviceBuffer(a.nbytes)
        d_in.upload(a)
        _lib.synchronize()
        lengths, total = np.zeros(len(sel), np.int64), C.c_int64()
        before = L.fa_kernel_launch_count()
        _lib.check(L.fa_luxtts_finish_device(dev._h, len(sel), ds.ctypes.data, d_in.ptr, 290000, 290000, d_out.ptr,
                                             a.size, lengths.ctypes.data, C.byref(total)), "fin")
        assert L.fa_kernel_launch_count() - before == 1
        _lib.synchronize()
        assert d_out.download(total.value, np.float32).tobytes() == np.concatenate(want).tobytes()
    host.close_handle()
    dev.close_handle()


# ------------------------------------------------------------------------------------------------ end to end
def test_synthesize_batch_equals_the_oracle(mel):
    rng = np.random.default_rng(7)
    prompts, pt, tt, speeds, _ = _begin_case(rng, 6)
    speeds[:] = np.float32(1.0)
    ptok = [list(rng.integers(1, 120, size=a)) for a in pt]
    ttok = [list(rng.integers(1, 120, size=b)) for b in tt]
    table = rng.normal(size=(128, 112)).astype(np.float32)

    def text_encoder(tokens, mask):
        return (table[tokens] * (1 - mask[..., None])).astype(np.float32)

    def fm_decoder(t, x, tc, sc, g, pm):
        return (np.float32(0.5) * x + tc - sc + t.reshape(-1, 1, 1)).astype(np.float32)

    def vocoder(m):
        b = m.shape[-1]
        return np.tanh(np.repeat(m.mean(axis=1), 512, axis=-1)[:, :(b - 1) * 512] * np.float32(3)).astype(np.float32)

    got = LX.LuxTtsSynthesizer(text_encoder, fm_decoder, vocoder).synthesize_batch(ptok, ttok, prompts, 1.0, 42)
    for i, res in enumerate(got):
        want = O.synthesize(ptok[i], ttok[i], prompts[i], 1.0, 42, lambda a, b: text_encoder(a, b),
                            lambda *a: fm_decoder(*a)[..., :100], vocoder, mel.extract)
        samples, P, G, L = want
        assert (res.prompt_frames, res.generated_frames, res.features_length) == (P, G, L)
        assert res.samples.tobytes() == samples.tobytes(), i


# ------------------------------------------------------------------------------------------------ fixture
def test_the_reference_fixture(mel):
    with open(os.path.join(GOLDEN, "luxtts_fixtures.json")) as f:
        fx = json.load(f)
    audio = np.fromfile(os.path.join(GOLDEN, "prompt_24k_f32le.bin"), np.float32)
    ref = np.fromfile(os.path.join(GOLDEN, "prompt_mel_f32le.bin"), np.float32).reshape(-1, 100)
    m = mel.extract(audio)
    assert m.shape == (406, 100) == ref.shape
    assert np.abs(m * np.float32(0.1) - ref).max() < 1e-3
    pt = len(fx["prompt"]["token_ids"])
    got = [LX.plan(audio.size, pt, len(t["token_ids"]), 1.0) for t in fx["texts"]]
    assert [p.features_length for p in got] == [838, 868] and {p.bucket for p in got} == {555}
    R = LX.LuxTtsRequests()
    _, plans, _, _ = R.begin([audio], [pt], [len(fx["texts"][0]["token_ids"])], [1.0], [42])
    want = np.float32(fx["prompt"]["rms_pre_norm"])
    assert abs(int(np.float32(plans[0].prompt_rms).view(np.int32)) - int(want.view(np.int32))) <= 1
    assert plans[0].gen_frames == fx["e2e"]["gen_frames"]
    R.close_handle()
