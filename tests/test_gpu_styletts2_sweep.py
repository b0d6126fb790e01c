"""StyleTTS2 synthesis glue on the H100 against the oracle (oracle/oracle_styletts2.cpp): sampler inputs for 1 … 1 024
requests in every bucket, the style blend with edge weights and non-finite inputs, align across logit widths, channel
counts that hit tile edges, F from 1 to over 12 000 and two frame strides, its refusals, host against device variants
with their launch counts, and synthesize_batch with deterministic fake models against the oracle's synthesize."""
import ctypes as C
import math

import numpy as np
import pytest

from fluidaudio_b200 import _lib
from fluidaudio_b200 import styletts2 as S
from oracle import oracle_styletts2 as O

pytestmark = pytest.mark.gpu

MASK = (1 << 64) - 1
GAMMA = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module", autouse=True)
def device():
    if _lib.device_count() < 1:
        pytest.skip("needs an H100")
    _lib.set_device(0)


@pytest.fixture(scope="module")
def glue():
    return S.StyleTTS2Glue()


def _uniform(s0, k):
    z = (s0 + k * GAMMA) & MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
    z ^= z >> 31
    u = float(z >> 11) / float(1 << 53)
    return u if u > 0 else 2.2250738585072014e-308


def _near_midpoint(v):
    """v (float64) lies within 2^-40 (relative) of a float32 rounding midpoint"""
    f = np.float32(v)
    other = np.nextafter(f, np.float32(np.inf) if float(f) < v else np.float32(-np.inf))
    mid = (float(f) + float(other)) / 2
    return abs(v - mid) <= 2.0 ** -40 * abs(v)


def _noise_exceptions(got, want, seed):
    """positions where got != want; each must be the float32 neighbour of a float64 value near a midpoint"""
    s0 = 0xdeadbeefcafebabe if seed == 0 else seed
    bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
    for j in bad.tolist():
        d = math.sqrt(-2.0 * math.log(_uniform(s0, 2 * j + 1))) * math.cos(2.0 * math.pi * _uniform(s0, 2 * j + 2))
        assert abs(int(got[j:j + 1].view(np.int32)[0]) - int(want[j:j + 1].view(np.int32)[0])) == 1, j
        assert _near_midpoint(d), (j, d)
    return bad.size


def _duration_exceptions(got, want, logits):
    """tokens whose duration differs; each must differ by one and hold an exp value near a float32 midpoint"""
    bad = np.flatnonzero(np.asarray(got) != np.asarray(want))
    for t in bad.tolist():
        assert abs(int(got[t]) - int(want[t])) == 1, t
        assert any(_near_midpoint(math.exp(-float(x))) for x in logits[t] if abs(float(x)) < 80), t
    return bad.size


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and np.array_equal(np.where(both, 0, a).view(np.int32), np.where(both, 0, b).view(np.int32))


# ------------------------------------------------------------------------------------------------ sampler inputs
@pytest.mark.parametrize("n", [1, 3, 64, 1024])
@pytest.mark.parametrize("bucket", [57, 64, 128, 256])
def test_sampler_inputs_equal_the_oracle(glue, n, bucket):
    rng = np.random.default_rng(n * 1000 + bucket)
    lo = {57: 1, 64: 58, 128: 65, 256: 129}[bucket]
    sizes = rng.integers(lo, bucket + 1, size=n)
    sizes[0] = bucket
    ids = [rng.integers(0, 178, size=k).astype(np.int32) for k in sizes]
    seeds = rng.integers(0, 2**63, size=n).astype(np.uint64)
    seeds[0] = 0
    tokens, mask, noise = glue.sampler_inputs(ids, seeds, bucket)
    exceptions = 0
    for i in range(n):
        t, m, ni, na = O.sampler_inputs(ids[i], bucket, int(seeds[i]))
        assert tokens[i].tobytes() == t.tobytes() and mask[i].tobytes() == m.tobytes()
        exceptions += _noise_exceptions(noise[i].reshape(-1), np.concatenate([ni, na.reshape(-1)]), int(seeds[i]))
    print(f"bucket {bucket}, {n} requests: {exceptions} noise exceptions over {n * 1280} Gaussians")


# ------------------------------------------------------------------------------------------------ style
def test_style_bit_for_bit(glue):
    rng = np.random.default_rng(11)
    n = 300
    p, r = rng.normal(size=(n, 256)).astype(np.float32), rng.normal(size=(n, 256)).astype(np.float32) * 3
    special = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 3.4e38, -3.4e38, 1e-45], np.float32)
    p.reshape(-1)[rng.choice(p.size, 200, replace=False)] = rng.choice(special, 200)
    r.reshape(-1)[rng.choice(r.size, 200, replace=False)] = rng.choice(special, 200)
    a = rng.uniform(-0.5, 1.5, size=n).astype(np.float32)
    b = rng.uniform(-0.5, 1.5, size=n).astype(np.float32)
    a[:4], b[:4] = [1.0, 0.0, 0.3, np.nan], [0.0, 1.0, 0.7, np.inf]
    ref, s = glue.blend_style(p, r, a, b)
    for i in range(n):
        wr, ws = O.blend(p[i], r[i], a[i], b[i])
        assert _bits_equal(ref[i], wr) and _bits_equal(s[i], ws), i


# ------------------------------------------------------------------------------------------------ align
def _logits(rng, durations, C_):
    """logits [n x C] whose sigmoid sums are near the wanted durations, plus noise"""
    n = len(durations)
    x = np.where(np.arange(C_)[None, :] < np.asarray(durations)[:, None], 30.0, -30.0)
    return (x + rng.normal(size=(n, C_)) * 2).astype(np.float32)


def _align_case(rng, counts, C_, dC, tC, long=False):
    logits, d, t_en = [], [], []
    for n in counts:
        dur = np.full(n, C_) if long else rng.integers(1, min(C_, 9) + 1, size=n)
        lg = _logits(rng, dur, C_) if C_ > 1 else rng.normal(size=(n, 1)).astype(np.float32) * 4
        logits.append(lg)
        d.append(rng.normal(size=(n, dC)).astype(np.float32))
        t_en.append(rng.normal(size=(tC, n)).astype(np.float32))
    return logits, d, t_en


@pytest.mark.parametrize("C_", [1, 4, 50])
@pytest.mark.parametrize("dC,tC", [(640, 512), (3, 33), (33, 3)])
def test_align_equals_the_oracle(glue, C_, dC, tC):
    rng = np.random.default_rng(C_ * 7 + dC)
    counts = [1, 2, 57, 100, 256, 31]
    logits, d, t_en = _align_case(rng, counts, C_, dC, tC)
    # -0, inf and NaN in d and t_en reach only their own token's frames
    special = np.array([np.nan, np.inf, -np.inf, -0.0], np.float32)
    for a in d[3:4] + t_en[3:4]:
        a.reshape(-1)[rng.choice(a.size, 8, replace=False)] = rng.choice(special, 8)
    want = [O.align(lg, dd, tt) for lg, dd, tt in zip(logits, d, t_en)]
    top = max(w[1] for w in want)
    exceptions = 0
    for stride in (top, top + 77):
        en, asr, frames, durations = glue.align(logits, d, t_en, frame_stride=stride)
        for i, (dur, F, wen, wasr) in enumerate(want):
            exceptions += _duration_exceptions(durations[i], dur, logits[i])
            if (durations[i] == dur).all():
                assert frames[i] == F
                assert _bits_equal(en[i, :, :F], wen) and _bits_equal(asr[i, :, :F], wasr), i
                assert not en[i, :, F:].any() and not asr[i, :, F:].any()
    print(f"C={C_} dC={dC} tC={tC}: frames {[w[1] for w in want]}, {exceptions} duration exceptions")


def test_align_long_and_single_frame(glue):
    rng = np.random.default_rng(21)
    logits, d, t_en = _align_case(rng, [256, 256], 50, 640, 512, long=True)   # every token 50 frames: F = 12 800
    lg1 = np.full((1, 1), -40.0, np.float32)                                   # one token, one frame: F = 1
    logits.append(lg1)
    d.append(rng.normal(size=(1, 640)).astype(np.float32))
    t_en.append(rng.normal(size=(512, 1)).astype(np.float32))
    logits = [np.pad(x, ((0, 0), (0, 50 - x.shape[1])), constant_values=-40.0) for x in logits]
    en, asr, frames, durations = glue.align(logits, d, t_en)
    assert frames.tolist()[2] == 1 and frames.max() > 12000
    for i in range(3):
        dur, F, wen, wasr = O.align(logits[i], d[i], t_en[i])
        assert (durations[i] == dur).all() and frames[i] == F
        assert _bits_equal(en[i, :, :F], wen) and _bits_equal(asr[i, :, :F], wasr)
        assert not en[i, :, F:].any() and not asr[i, :, F:].any()


def _raw_align(L, counts, logits, C_, d, dC, t, tC, stride, device=False):
    counts = np.asarray(counts, np.int32)
    n, w = counts.size, int(counts.max())
    en, asr = np.full(n * dC * stride, 7, np.float32), np.full(n * tC * stride, 7, np.float32)
    frames, durs, reasons = np.full(n, -9, np.int64), np.full(int(counts.sum()), -9, np.int32), np.full(n, -9, np.int32)
    st = L.fa_styletts2_align(n, _lib.ptr(counts), _lib.ptr(logits), C_, C_, w * C_, _lib.ptr(d), dC, dC, w * dC,
                              _lib.ptr(t), tC, w, tC * w, stride, _lib.ptr(en), _lib.ptr(asr), _lib.ptr(frames),
                              _lib.ptr(durs), _lib.ptr(reasons))
    return st, en, asr, frames, durs, reasons


def test_align_refusals_write_nothing():
    L = _lib.load()
    rng = np.random.default_rng(31)
    counts = [5, 7]
    logits = np.zeros((2, 7, 4), np.float32)   # every token 2 frames: F = 10, 14
    d, t = rng.normal(size=(2, 7, 3)).astype(np.float32), rng.normal(size=(2, 2, 7)).astype(np.float32)
    st, en, asr, frames, durs, reasons = _raw_align(L, counts, logits, 4, d, 3, t, 2, 14)
    assert st == 0 and frames.tolist() == [10, 14] and (durs == 2).all() and (reasons == 0).all()
    st, en, asr, frames, durs, reasons = _raw_align(L, counts, logits, 4, d, 3, t, 2, 13)
    assert st == 3 and frames.tolist() == [10, 14] and (en == 7).all() and (asr == 7).all() and (durs == -9).all()
    assert b"frame_stride" in L.fa_last_error()
    bad = logits.copy()
    bad[1, 6, 3] = np.nan
    st, en, asr, frames, durs, reasons = _raw_align(L, counts, bad, 4, d, 3, t, 2, 14)
    assert st == 1 and reasons.tolist() == [0, 3] and (frames == -9).all() and (en == 7).all() and (durs == -9).all()
    assert b"NaN" in L.fa_last_error()
    bad[1, 6, 3] = 0
    bad[0, 5:, :] = np.nan   # past request 0's 5 tokens: never read
    st, *_ = _raw_align(L, counts, bad, 4, d, 3, t, 2, 14)
    assert st == 0


# ------------------------------------------------------------------------------------------------ host vs device
def test_device_variants_equal_host_variants_with_their_launch_counts(glue):
    rng = np.random.default_rng(41)
    L = _lib.load()
    n, bucket = 37, 128
    sizes = rng.integers(65, 129, size=n)
    ids = [rng.integers(0, 178, size=k).astype(np.int32) for k in sizes]
    seeds = rng.integers(0, 2**63, size=n).astype(np.uint64)
    before = _lib.kernel_launch_count()
    tokens, mask, noise = glue.sampler_inputs(ids, seeds, bucket)
    assert _lib.kernel_launch_count() - before == 1
    flat = np.concatenate(ids)
    d_ids = _lib.DeviceBuffer(flat.nbytes)
    d_ids.upload(flat)
    d_tok, d_mask, d_noise = (_lib.DeviceBuffer(tokens.nbytes), _lib.DeviceBuffer(mask.nbytes),
                              _lib.DeviceBuffer(noise.nbytes))
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    before = _lib.kernel_launch_count()
    glue.sampler_inputs_device(n, d_ids.ptr, off, seeds, bucket, d_tok.ptr, d_mask.ptr, d_noise.ptr)
    assert _lib.kernel_launch_count() - before == 1
    _lib.synchronize()
    assert d_tok.download(tokens.shape, np.int32).tobytes() == tokens.tobytes()
    assert d_mask.download(mask.shape, np.int32).tobytes() == mask.tobytes()
    assert d_noise.download(noise.shape, np.float32).tobytes() == noise.tobytes()

    p, r = rng.normal(size=(n, 256)).astype(np.float32), rng.normal(size=(n, 256)).astype(np.float32)
    a, b = rng.uniform(size=n).astype(np.float32), rng.uniform(size=n).astype(np.float32)
    before = _lib.kernel_launch_count()
    ref, s = glue.blend_style(p, r, a, b)
    assert _lib.kernel_launch_count() - before == 1
    bufs = [_lib.DeviceBuffer(x.nbytes) for x in (p, r, ref, s)]
    bufs[0].upload(p)
    bufs[1].upload(r)
    before = _lib.kernel_launch_count()
    glue.blend_style_device(n, bufs[0].ptr, bufs[1].ptr, a, b, bufs[2].ptr, bufs[3].ptr)
    assert _lib.kernel_launch_count() - before == 1
    _lib.synchronize()
    assert bufs[2].download(ref.shape, np.float32).tobytes() == ref.tobytes()
    assert bufs[3].download(s.shape, np.float32).tobytes() == s.tobytes()

    counts = rng.integers(1, 120, size=n)
    logits, d, t_en = _align_case(rng, counts, 50, 640, 512)
    before = _lib.kernel_launch_count()
    en, asr, frames, durations = glue.align(logits, d, t_en, frame_stride=1200)
    assert _lib.kernel_launch_count() - before == 2
    w = int(counts.max())
    L_, D_, T_ = np.zeros((n, w, 50), np.float32), np.zeros((n, w, 640), np.float32), np.zeros((n, 512, w), np.float32)
    for i in range(n):
        k = counts[i]
        L_[i, :k], D_[i, :k], T_[i, :, :k] = logits[i], d[i], t_en[i]
    ins = [_lib.DeviceBuffer(x.nbytes) for x in (L_, D_, T_)]
    for buf, x in zip(ins, (L_, D_, T_)):
        buf.upload(x)
    d_en, d_asr = _lib.DeviceBuffer(en.nbytes), _lib.DeviceBuffer(asr.nbytes)
    before = _lib.kernel_launch_count()
    st, dframes, ddur, _ = glue.align_device(counts, ins[0].ptr, 50, 50, w * 50, ins[1].ptr, 640, 640, w * 640,
                                             ins[2].ptr, 512, w, 512 * w, 1200, d_en.ptr, d_asr.ptr)
    assert st == 0 and _lib.kernel_launch_count() - before == 2
    _lib.synchronize()
    assert (dframes == frames).all() and (ddur == np.concatenate(durations)).all()
    assert d_en.download(en.shape, np.float32).tobytes() == en.tobytes()
    assert d_asr.download(asr.shape, np.float32).tobytes() == asr.tobytes()
    before = _lib.kernel_launch_count()
    st, tframes, _, _ = glue.align_device(counts, ins[0].ptr, 50, 50, w * 50, ins[1].ptr, 640, 640, w * 640,
                                          ins[2].ptr, 512, w, 512 * w, int(frames.max()) - 1, d_en.ptr, d_asr.ptr)
    assert st == 3 and (tframes == frames).all() and _lib.kernel_launch_count() - before == 1
    for buf in [d_ids, d_tok, d_mask, d_noise, d_en, d_asr] + bufs + ins:
        buf.free()


# ------------------------------------------------------------------------------------------------ end to end
TC, DC, DEN, BERT, CL = 5, 7, 6, 16, 4


def text_encoder(tokens, lengths, mask):
    t = tokens.astype(np.float32)
    return np.sin(t[:, None, :] * np.float32(0.1) + np.arange(TC, dtype=np.float32)[None, :, None]).astype(np.float32)


def bert(tokens, mask):
    t = tokens.astype(np.float32)
    dur = np.cos(t[:, :, None] * np.float32(0.05) + np.arange(BERT, dtype=np.float32)).astype(np.float32)
    d_en = (np.cos(t[:, None, :] * np.float32(0.2) + np.arange(DEN, dtype=np.float32)[None, :, None]) *
            mask[:, None, :].astype(np.float32)).astype(np.float32)
    return dur, d_en


def ref_encoder(mel):
    m = mel.reshape(80, -1)
    return (np.resize(m.mean(axis=1), 256) + np.arange(256, dtype=np.float32) * np.float32(0.01)).astype(
        np.float32)[None]


def sampler(noise_init, noises_aux, embedding, features):
    k = features.shape[0]
    aux = noises_aux.reshape(k, 4, 256)
    out = (noise_init.reshape(k, 256) * np.float32(0.5) + (aux[:, 0] - aux[:, 3]) * np.float32(0.1)
           + features * np.float32(0.3) + embedding.reshape(k, -1)[:, :1])
    return out.astype(np.float32)[:, None, :]


def duration_predictor(d_en, s, mask):
    x = d_en[0].T   # [n x 6]
    d = np.concatenate([x, x[:, :1] * s[0, 0]], axis=1).astype(np.float32)[None]
    logits = (np.tile(x[:, :CL], 1) * np.float32(4) + s[0, :CL] - np.float32(1)).astype(np.float32)[None]
    return d, logits


def f0n_har(en, s):
    return en[:, 0] + en[:, 1], en[:, 2] * np.float32(0.5) + s[:, :1], np.repeat(en[:, :1, :], 3, axis=2)


def decoder_pre(asr, f0, n, ref):
    return np.repeat(np.concatenate([asr[:, :4] + f0[:, None], n[:, None] * ref[:, :1, None]], axis=1), 2,
                     axis=2).astype(np.float32)


def decoder_upsample(x_pre, ref, har):
    return (np.repeat(x_pre[:, 0] - x_pre[:, 4], 30, axis=1) + ref[:, :1]).astype(np.float32)


MODELS = (text_encoder, bert, ref_encoder, sampler, duration_predictor, f0n_har, decoder_pre, decoder_upsample)


def test_synthesize_batch_equals_the_oracle():
    rng = np.random.default_rng(51)
    sizes = [3, 57, 58, 64, 100, 200, 256, 1, 40, 130]
    ids = [rng.integers(1, 178, size=k).astype(np.int32) for k in sizes]
    mels = [rng.normal(size=(80, int(rng.integers(20, 200)))).astype(np.float32) for _ in range(4)]
    refs = [0, 1, 1, 2, 3, 0, 1, 2, 2, 2]
    seeds = np.array([0, 5, 5, 9, 2**63, 3, 5, 7, 7, 7], np.uint64)
    alphas = np.array([0.3] * 9 + [1.0], np.float32)
    betas = np.array([0.7] * 9 + [0.0], np.float32)
    syn = S.StyleTTS2Synthesizer(*MODELS)
    got = syn.synthesize_batch(ids, mels, seeds, alphas, betas, references=refs)
    want = [O.synthesize(ids[i], mels[refs[i]], alphas[i], betas[i], int(seeds[i]), *MODELS) for i in range(len(ids))]
    for i, (g, w) in enumerate(zip(got, want)):
        samples, F, durations = w
        assert g.frames == F and (g.durations == durations).all(), i
        assert g.samples.tobytes() == samples.tobytes(), i
    # a chunked utterance: requests 1, 2 and 6 share reference 1 and seed 5, concatenated in order
    utter = [0, 1, 1, 2, 3, 4, 1, 5, 5, 5]
    chunked = syn.synthesize_batch(ids, mels, seeds, alphas, betas, references=refs, utterances=utter)
    assert len(chunked) == 6
    assert chunked[1].samples.tobytes() == np.concatenate([want[1][0], want[2][0], want[6][0]]).tobytes()
    assert chunked[5].samples.tobytes() == np.concatenate([want[7][0], want[8][0], want[9][0]]).tobytes()
    with pytest.raises(S.StyleTTS2Error):
        syn.synthesize_batch([ids[0], np.zeros(257, np.int32)], mels[:2], 0, 0.3, 0.7)
    with pytest.raises(S.StyleTTS2Error):
        syn.synthesize_batch([ids[0], []], mels[:2], 0, 0.3, 0.7)
