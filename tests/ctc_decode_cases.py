"""Seeded inputs of the CTC decoding tests: log-prob rows (random, tie-heavy quantised, constant, with -inf columns,
and peaky log-softmax rows like a model's),
SentencePiece-like vocabularies over a small alphabet (word starts, continuations, the bare U+2581, empty and missing
pieces) and synthetic bigram LMs whose words those pieces spell."""
import numpy as np

B = "▁"


def rows(rng, T, V, kind="normal"):
    if kind == "normal":
        x = rng.normal(0, 3, size=(T, V))
    elif kind == "ties":
        x = np.round(rng.normal(0, 1, size=(T, V)) * 2) / 2 - 3
    elif kind == "constant":
        x = np.full((T, V), -2.0)
    else:   # some -inf columns
        x = rng.normal(0, 3, size=(T, V))
        x[rng.random((T, V)) < 0.3] = -np.inf
    return x.astype(np.float32)


def vocabulary(rng, V, letters="abcdefgh", missing=0.05):
    """{id: piece} for ids 0 .. V-1, a few left out; id 0 is the bare U+2581 and id 1 the empty piece"""
    voc = {}
    for v in range(V):
        if v > 1 and rng.random() < missing:
            continue
        n = int(rng.integers(1, 3))
        core = "".join(rng.choice(list(letters), size=n))
        voc[v] = B if v == 0 else "" if v == 1 else (B + core if rng.random() < 0.4 else core)
    return voc


def pieces(voc, V):
    return [voc.get(v) for v in range(V)]


def synthetic_lm(rng, words=400, bigrams=2000, letters="abcdefgh", max_len=4):
    """unigrams {word: (log_prob, backoff)} and bigrams {context: {word: log_prob}}, natural log, float32; a tenth of the
    words appear in bigrams only"""
    vocab = set()
    while len(vocab) < words:
        vocab.add("".join(rng.choice(list(letters), size=int(rng.integers(1, max_len + 1)))))
    vocab = sorted(vocab)
    rng.shuffle(vocab)
    uni = {w: (np.float32(-rng.uniform(0.5, 8)), np.float32(-rng.uniform(0, 2))) for w in vocab[: int(words * 0.9)]}
    bi = {}
    for _ in range(bigrams):
        c, w = vocab[int(rng.integers(words))], vocab[int(rng.integers(words))]
        bi.setdefault(c, {})[w] = np.float32(-rng.uniform(0.1, 5))
    return uni, bi


def peaky(rng, T, V, sharpness=8.0, blank=None):
    """[T x V] float32 log-softmax of logits shaped like a CTC model's output: runs of blank frames between tokens held
    for one to three frames, each frame's mass almost all on its dominant column (logit lead `sharpness` over unit
    normal noise).  With the blank outside [0, V) a blank run has no dominant column."""
    blank = V - 1 if blank is None else blank
    tokens = [v for v in range(V) if v != blank]
    x = rng.normal(0, 1, size=(T, V))
    t = 0
    while t < T:
        n = int(rng.geometric(0.3))
        if 0 <= blank < V:
            x[t:t + n, blank] += sharpness
        t += n
        if tokens:
            n = int(rng.integers(1, 4))
            x[t:t + n, tokens[int(rng.integers(len(tokens)))]] += sharpness
            t += n
    x -= x.max(1, keepdims=True)
    return (x - np.log(np.exp(x).sum(1, keepdims=True))).astype(np.float32)
