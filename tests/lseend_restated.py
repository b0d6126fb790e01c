"""LSEENDFeatureProvider and StreamingChunkQueue (Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384) restated in plain
Python and numpy float32, independently of ``oracle/oracle_lseend.cpp``: the same provider with the log-mel passed in,
so that the CPU tests can pin the oracle's queues, running mean, mask and snapshots to it, and the GPU tests can run the
reference's own buffer construction over the library's ``fa_mel_lseend_features``."""
import math

import numpy as np

F32 = np.float32
SCALE = F32(1.0) / F32(math.log(10.0))   # :36, 1 / logf(10) in float32


def derived(cfg):
    """(n_fft, mel_frames, chunk_mels, chunk_samples, flush_samples) of LSEENDMetadata (LSEENDTypes.swift:53-57) and
    the provider's init (:52-61)."""
    n_fft = 1 << (cfg["win_length"] - 1).bit_length()
    sub, chunk, ctx, hop = cfg["subsampling"], cfg["chunk_size"], cfg["context_size"], cfg["hop_length"]
    return (n_fft, (chunk - 1) * sub + 2 * ctx + 1, sub * chunk, hop * sub * chunk,
            (ctx + cfg["conv_delay"] * sub) * hop + n_fft // 2)


class Queue:
    """StreamingChunkQueue (:284-384) over rows of `stride` floats, kept as a flat list of float32 values."""

    def __init__(self, chunk_length, left, right, stride):
        self.stride = stride
        self.chunk = chunk_length * stride
        self.context = (left + right) * stride
        self.padded = self.chunk + self.context
        self.left = left * stride
        self.reset()

    def reset(self):
        self.buf = np.zeros(self.left, F32)
        self.head = 0

    def copy(self):
        q = Queue.__new__(Queue)
        q.__dict__.update(self.__dict__)
        q.buf = self.buf.copy()
        return q

    @property
    def unread(self):
        return self.buf.size - self.head

    @property
    def ready(self):
        return max(0, (self.unread - self.context) // self.chunk)

    def has_chunk(self):
        return self.unread >= self.padded

    def append(self, x):
        self.buf = np.concatenate([self.buf, np.asarray(x, F32).reshape(-1)])

    def pop_next(self):
        if not self.has_chunk():
            return None
        out = self.buf[self.head:self.head + self.padded].copy()
        self.head += self.chunk
        return out

    def pop_all(self):
        if not self.has_chunk():
            return None
        new_head = self.head + (self.buf.size - self.head - self.context) // self.chunk * self.chunk
        out = self.buf[self.head:new_head + self.context].copy()
        self.head = new_head
        return out


def scale_cmn(x, mean, count):
    """:259-276 in numpy float32, frames in order: v = x * scale; mean += alpha * (v - mean); x = v - mean."""
    x = np.asarray(x, F32).copy()
    mean = np.asarray(mean, F32).copy()
    with np.errstate(all="ignore"):
        for t in range(x.shape[0]):
            count += 1
            alpha = F32(1.0) / F32(count)
            v = (x[t] * SCALE).astype(F32)
            mean = (mean + (alpha * (v - mean).astype(F32)).astype(F32)).astype(F32)
            x[t] = (v - mean).astype(F32)
    return x, mean, count


class Provider:
    """The provider.  ``features(slice, mean, count) -> (rows [T x nMels], mean', count')`` is processAudioQueue's
    log-mel, scaling and running mean of one popAllChunks slice; by default a .prePadded log-mel ``mel(slice)`` followed
    by ``scale_cmn``."""

    def __init__(self, cfg, mel=None, features=None):
        self.cfg = cfg
        n_fft, self.mel_frames, chunk_mels, chunk_samples, self.flush = derived(cfg)
        hop, ctx, M = cfg["hop_length"], cfg["context_size"], cfg["n_mels"]
        self.M, self.chunk_size = M, cfg["chunk_size"]
        self.mask = np.array([0.0] * cfg["conv_delay"] + [1.0] * cfg["chunk_size"], F32)
        self.features = features or (lambda s, mean, count: scale_cmn(mel(s), mean, count))
        self.mel_q = Queue(chunk_mels, ctx, ctx + 1 - cfg["subsampling"], M)
        self.audio_q = Queue(chunk_samples, n_fft // 2, n_fft // 2 - hop, 1)
        self.slices = []   # every popAllChunks slice, in order
        self.reset()

    def reset(self):
        self.mel_q.reset()
        self.audio_q.reset()
        self.mean, self.count, self.mask_end = np.zeros(self.M, F32), 0, 0

    def _process(self):
        s = self.audio_q.pop_all()
        if s is None:
            return
        self.slices.append(s)
        rows, self.mean, self.count = self.features(s, self.mean, self.count)
        self.mel_q.append(rows)

    def enqueue_audio(self, x):
        self.audio_q.append(x)
        self._process()

    def drain_right_context_with_silence(self):
        q = self.audio_q
        q.append(np.zeros(self.flush, F32))
        over = max(0, q.unread - q.context)
        q.append(np.zeros((q.chunk - over % q.chunk) % q.chunk, F32))
        self._process()

    def emit_next_chunk(self):
        self._process()
        raw = self.mel_q.pop_next()
        if raw is None:
            return None
        self.mask_end = min(self.mask_end + self.chunk_size, self.mask.size)
        return (raw.reshape(self.mel_frames, self.M), self.mask[self.mask_end - self.chunk_size:self.mask_end].copy(),
                min(self.mask.size - self.mask_end, self.chunk_size))

    def push(self, x, drain=False):
        self.enqueue_audio(x)
        if drain:
            self.drain_right_context_with_silence()
        out = []
        while (c := self.emit_next_chunk()) is not None:
            out.append(c)
        f = np.stack([c[0] for c in out]) if out else np.zeros((0, self.mel_frames, self.M), F32)
        m = np.stack([c[1] for c in out]) if out else np.zeros((0, self.chunk_size), F32)
        return f, m, np.array([c[2] for c in out], np.int32)

    def take_snapshot(self):
        return (self.mel_q.copy(), self.audio_q.copy(), self.mean.copy(), self.count, self.mask_end)

    def rollback(self, snap):
        mq, aq, mean, count, end = snap
        self.mel_q, self.audio_q, self.mean, self.count, self.mask_end = mq.copy(), aq.copy(), mean.copy(), count, end

    def state(self):
        return dict(audio=self.audio_q.buf[self.audio_q.head:].copy(),
                    mel=self.mel_q.buf[self.mel_q.head:].reshape(-1, self.M).copy(), cmn_mean=self.mean.copy(),
                    cmn_count=self.count, decoder_mask_end=self.mask_end)


def push_sequence(rng, chunk_samples, hop, steps):
    """Seeded push sizes and drain flags: empty pushes, pushes below one hop, around one chunk, many chunks, and drains
    followed by more audio."""
    out = []
    for _ in range(steps):
        kind = int(rng.integers(0, 6))
        n = (0, int(rng.integers(1, hop)) if hop > 1 else 1, int(rng.integers(1, 2 * chunk_samples)),
             int(rng.integers(3, 6)) * chunk_samples + int(rng.integers(0, chunk_samples)),
             int(rng.integers(0, chunk_samples // 2 + 1)), chunk_samples)[kind]
        out.append((n, bool(rng.random() < 0.15)))
    return out
