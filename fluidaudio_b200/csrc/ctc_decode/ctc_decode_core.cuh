// Host- and device-callable arithmetic of CTC decoding (ctc_decode_kernels.cu; its host build is tests/emul/
// ctc_decode_emul.cpp): ctcGreedyDecode and ctcBeamSearch (CtcDecoder.swift:15-70, :118-277), logAddExp
// (:282-287) and ARPALanguageModel.score (ARPALanguageModel.swift:92-96), one frame's candidates at a time.  Every float
// operation is one fa::fp helper, and exp is ctc_core.cuh's, so the kernels and the host build compute the same bits.
//
// The beam search in the kernels' formulation.  Beam i of the frame's nb beams (in contract order) owns candidate slots
// i * (K + 1) + c: c = 0 is its keep candidate (the blank extension, its repeat-same and, when its parent prefix is also
// a beam of the frame and its last token one of the K candidate tokens, the parent's extension folded in), c >= 1 the
// extension by the frame's candidate token c - 1.  A slot's generation index is its position in the reference's
// insertion order; a keep whose parent's extension comes first takes that extension's index, and the extension slot
// is dead.  The prune keeps the beam_width smallest order keys (total descending, generation index ascending), in
// that order.  Prefixes are nodes of a per-clip hash-consed trie (cons), so node equality is prefix equality.
#pragma once

#include "../ctc/ctc_core.cuh"

#include <cstdint>

namespace fa {
namespace ctc_decode {

constexpr int kMaxBeamWidth = 128;        // FA_CTC_DECODE_MAX_BEAM_WIDTH
constexpr int kMaxTokenCandidates = 64;   // FA_CTC_DECODE_MAX_TOKEN_CANDIDATES
constexpr float kUnkLogProb = -23.026f;   // ARPALanguageModel.unkLogProb
constexpr int kNoToken = -1;              // the last token of the empty prefix
constexpr int kRootNode = 0;              // the empty prefix
constexpr int kLmRoot = 0;                // the empty partial word
constexpr int kLmDead = -1;               // a non-empty partial word that starts no LM word
constexpr int kNoWord = -1;               // prevWord nil, or a word the LM does not know (the same thing to score)
constexpr unsigned long long kEmpty = ~0ull;   // an empty hash slot, and the order key of a dead candidate slot

// logAddExp: b when a is -inf, a when b is, else m + log(exp(a - m) + exp(b - m)) with m = Swift.max(a, b)
FA_HD float log_add_exp(float a, float b) {
    using namespace fp;
    if (a == -INFINITY) return b;
    if (b == -INFINITY) return a;
    const float m = swift_max(a, b);
    return f_add(m, f_log(f_add(f_exp(f_sub(a, m)), f_exp(f_sub(b, m)))));
}

// CtcBeam.total: totalAcoustic + lmScore
FA_HD float beam_total(float pb, float pnb, float lm) { return fp::f_add(log_add_exp(pb, pnb), lm); }

// The candidate tokens of a frame: every column but the blank, value descending, ties to the lower index.  True when
// column (va, ia) comes before column (vb, ib).
FA_HD bool ranks_before(float va, int ia, float vb, int ib) { return va > vb || (!(vb > va) && ia < ib); }

// ctcGreedyDecode's argmax as a fold: (vb, ib) replaces (va, ia) when it is strictly greater, or equal at a lower
// index (the first maximum); a NaN never replaces.  Column 0 as NaN wins outright (the caller checks it).
FA_HD bool greedy_better(float vb, int ib, float va, int ia) { return vb > va || (vb == va && ib < ia); }

// A frame's id is kept when it is not the blank and differs from the previous frame's id (blank included).
FA_HD bool greedy_keep(int id, int prev, int blank) { return id != blank && id != prev; }

// The order key of a candidate slot: the float order of -total in the high word (-0 and +0 tie, as Swift's > has
// them), then the generation index, then the slot index as payload.  Smaller keys come first.
FA_HD unsigned long long order_key(float total, int gen, int slot) {
    unsigned u;
    const float t = total == 0.0f ? 0.0f : total;
#if defined(__CUDA_ARCH__)
    u = __float_as_uint(t);
#else
    __builtin_memcpy(&u, &t, 4);
#endif
    const unsigned asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)~asc << 32) | ((unsigned long long)gen << 14) | (unsigned long long)slot;
}
FA_HD int key_slot(unsigned long long key) { return (int)(key & 0x3fff); }

// 64-bit mix of a hash key (the splitmix64 finaliser)
FA_HD unsigned long long mix(unsigned long long x) {
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// The home slot of `key` in a table of `cap` slots (cap < 2^32: a 32-bit remainder)
FA_HD long long home_slot(unsigned long long key, long long cap) {
    return (long long)((unsigned)(mix(key) >> 32) % (unsigned)cap);
}

// ------------------------------------------------------------------------------------------------ the prefix trie
// A clip's prefixes: node n >= 1 is hash slot n - 1 of an open-addressing table of `cap` keys (parent << 32 | token),
// so a node is found before it is made, and the table is the node store.  cas(slot, expected, desired) returns the
// slot's old key (atomicCAS on the device).
FA_HD unsigned long long trie_key(int parent, int token) {
    return ((unsigned long long)(unsigned)parent << 32) | (unsigned)token;
}
template <typename Cas> FA_HD int cons(unsigned long long *keys, long long cap, int parent, int token, Cas cas) {
    const unsigned long long k = trie_key(parent, token);
    long long s = home_slot(k, cap);
    for (;;) {
        const unsigned long long old = keys[s] == kEmpty ? cas(s, kEmpty, k) : keys[s];
        if (old == kEmpty || old == k) return (int)(s + 1);
        s = s + 1 == cap ? 0 : s + 1;
    }
}
FA_HD int node_parent(const unsigned long long *keys, int node) { return (int)(keys[node - 1] >> 32); }
FA_HD int node_token(const unsigned long long *keys, int node) { return (int)(unsigned)keys[node - 1]; }

// ------------------------------------------------------------------------------------------------ the language model
// ARPALanguageModel in HBM: a byte trie over every word it names (node 0 the empty word; children in an open-addressing
// table of (node << 8 | byte) keys), each node's word (kNoWord when it ends none), the unigram log-prob (unkLogProb
// when the word has none) and backoff (0 when none) per word, and the bigrams in an open-addressing table of
// (context << 32 | word) keys.
struct LmView {
    const unsigned long long *child_key;
    const int *child_node;
    long long child_cap;
    const int *node_word;
    const float *uni_log_prob, *uni_backoff;
    const unsigned long long *bigram_key;
    const float *bigram_log_prob;
    long long bigram_cap;
};

FA_HD int lm_child(const LmView &lm, int node, unsigned char byte) {
    const unsigned long long k = ((unsigned long long)(unsigned)node << 8) | byte;
    for (long long s = home_slot(k, lm.child_cap);; s = s + 1 == lm.child_cap ? 0 : s + 1) {
        const unsigned long long x = lm.child_key[s];
        if (x == k) return lm.child_node[s];
        if (x == kEmpty) return kLmDead;
    }
}

// The partial word `state` with the bytes p[0 .. n) appended
FA_HD int lm_walk(const LmView &lm, int state, const unsigned char *p, long long n) {
    for (long long i = 0; i < n && state != kLmDead; ++i) state = lm_child(lm, state, p[i]);
    return state;
}

// The word a non-empty partial word is: an LM word, or kNoWord (not a prefix of any, or a prefix that ends none)
FA_HD int lm_word(const LmView &lm, int state) { return state == kLmDead ? kNoWord : lm.node_word[state]; }

// score(word, prev): the bigram [prev][word] when there is one, else backoff(prev) + logProb(word)
FA_HD float lm_score(const LmView &lm, int word, int prev) {
    if (prev != kNoWord && word != kNoWord) {
        const unsigned long long k = ((unsigned long long)(unsigned)prev << 32) | (unsigned)word;
        for (long long s = home_slot(k, lm.bigram_cap);;
             s = s + 1 == lm.bigram_cap ? 0 : s + 1) {
            const unsigned long long x = lm.bigram_key[s];
            if (x == k) return lm.bigram_log_prob[s];
            if (x == kEmpty) break;
        }
    }
    const float backoff = prev != kNoWord ? lm.uni_backoff[prev] : 0.0f;
    return fp::f_add(backoff, word != kNoWord ? lm.uni_log_prob[word] : kUnkLogProb);
}

// lmWeight * score + wordBonus for the completed partial word `state` after `prev`
FA_HD float lm_delta(const LmView &lm, int state, int prev, float weight, float bonus) {
    return fp::f_add(fp::f_mul(weight, lm_score(lm, lm_word(lm, state), prev)), bonus);
}

// ------------------------------------------------------------------------------------------------ pieces
// The decoder's piece table: token v's bytes p[off[v] .. off[v+1]), boundary[v] when they start with U+2581, whose
// three bytes the word walk then skips (dropFirst).  An id the vocabulary lacks has the empty piece.
struct Pieces {
    const unsigned char *bytes;
    const long long *off;
    const unsigned char *boundary;
};

// ------------------------------------------------------------------------------------------------ one beam
struct Beam {
    float pb, pnb, lm;
    int node, parent, last, len;
    int word, prev;   // the partial word (LM trie state) and prevWord; untracked without an LM
};

// What a beam's extensions share in a frame: its acoustic total and, with an LM, what a word-boundary piece does
// (the LM delta is the parent's alone, so it is computed once per beam per frame).
struct Prelude {
    float total;        // totalAcoustic
    float delta;        // lmDelta of a boundary extension (0 without an LM or without a completed word)
    int prev;           // newPrevWord of a boundary extension
};
FA_HD Prelude prelude(const Beam &b, const LmView *lm, float weight, float bonus) {
    Prelude p{log_add_exp(b.pb, b.pnb), 0.0f, b.prev};
    if (lm && b.word != kLmRoot) {
        p.delta = lm_delta(*lm, b.word, b.prev, weight, bonus);
        p.prev = lm_word(*lm, b.word);
    }
    return p;
}

// The extension of b by v (log-prob lp): pNonBlank and lmScore; pBlank is -inf
FA_HD float ext_pnb(const Beam &b, const Prelude &p, int v, float lp) {
    return fp::f_add(b.last == v ? b.pb : p.total, lp);
}
FA_HD float ext_lm(const Beam &b, const Prelude &p, bool boundary) {
    return fp::f_add(b.lm, boundary ? p.delta : 0.0f);
}

// The keep candidate before any parent extension is folded in: the blank extension, then the repeat-same when v_rep
// (the last token's candidate log-prob) is present
FA_HD void keep_start(const Beam &b, const Prelude &p, float blank_lp, bool has_rep, float rep_lp, float &pb,
                      float &pnb) {
    pb = fp::f_add(p.total, blank_lp);
    pnb = has_rep ? log_add_exp(-INFINITY, fp::f_add(b.pnb, rep_lp)) : -INFINITY;
}

// The beam an extension of `b` by token v becomes, all but its node (cons) and probabilities
FA_HD Beam ext_beam(const Beam &b, const Prelude &p, int v, float pnb, const LmView *lm, const Pieces &pc) {
    Beam n = b;
    n.pb = -INFINITY;
    n.pnb = pnb;
    n.parent = b.node;
    n.last = v;
    n.len = b.len + 1;
    const bool boundary = pc.boundary[v] != 0;
    n.lm = ext_lm(b, p, boundary);
    if (lm) {
        const unsigned char *s = pc.bytes + pc.off[v];
        const long long k = pc.off[v + 1] - pc.off[v];
        if (boundary) {
            n.prev = p.prev;
            n.word = lm_walk(*lm, kLmRoot, s + 3, k - 3);
        } else {
            n.word = lm_walk(*lm, b.word, s, k);
        }
    }
    return n;
}

// The trailing partial word scored at the end, then the total
FA_HD float final_total(const Beam &b, const LmView *lm, float weight, float bonus) {
    const float lms = lm && b.word != kLmRoot ? fp::f_add(b.lm, lm_delta(*lm, b.word, b.prev, weight, bonus)) : b.lm;
    return beam_total(b.pb, b.pnb, lms);
}

} // namespace ctc_decode
} // namespace fa
