// CTC decoding on the GPU (ctc_decode_core.cuh holds the arithmetic):
//
//   topk_kernel     one warp per row of every clip: the frame's candidate tokens (value descending, index ascending,
//                   the blank left out), the blank's log-prob, and the lowest clip with a NaN or +inf in a row
//   beam_kernel     one CTA per clip: the prefix beam search over the clip's frames, its beams in shared memory in
//                   contract order.  Per frame: each beam's prelude, the extension slots' order keys, the keep slots
//                   (with the parent extensions folded in), a radix select of the beam_width smallest keys, their
//                   order, and the survivors' states (new prefixes consed into the clip's trie, the LM trie walked).
//                   At the end the trailing words are scored, the first best beam is backtraced into the clip's
//                   staging row.
//   argmax_kernel   one warp per row: ctcGreedyDecode's argmax
//   collapse_kernel one CTA per clip: the kept ids (not blank, not the previous frame's id) staged in order
//   gather_kernel   one CTA per clip: its staged tokens to their offset in the output
//
// A clip's frames are a dependent chain: one long clip is one CTA walking it, whatever the GPU's width.
#include "ctc_decode.h"

#include <algorithm>
#include <climits>
#include <cstring>

namespace fa {
namespace ctc_decode {

namespace {

constexpr int kWarps = 8;          // rows per CTA of topk_kernel / argmax_kernel
constexpr int kThreads = 256;      // beam_kernel, collapse_kernel, gather_kernel
constexpr int kTable = 256;        // node -> beam slots of a frame (at most 128 beams)
constexpr unsigned kFull = 0xffffffffu;
constexpr int kNoBad = 0x7f7f7f7f;   // the refusal flag as a byte fill leaves it: no clip is refused

// the clip whose rows include `row` (offs: clips + 1 offsets)
__device__ int clip_of(const long long *offs, int clips, long long row) {
    int lo = 0, hi = clips;   // offs[lo] <= row < offs[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (offs[mid] <= row) lo = mid;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kWarps * 32) topk_kernel(const float *__restrict__ lp, long long rows, int V,
                                                            int blank, int K, const long long *__restrict__ offs,
                                                            int clips, int *__restrict__ top_id,
                                                            float *__restrict__ top_lp, float *__restrict__ blank_lp,
                                                            int *__restrict__ bad) {
    const long long row = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float *x = lp + row * V;
    bool nonfinite = false;
    for (int v = lane; v < V; v += 32) {
        const float f = __ldg(x + v);
        nonfinite |= isnan(f) || f == INFINITY;
    }
    if (__any_sync(kFull, nonfinite)) {
        if (lane == 0) atomicMin(bad, clip_of(offs, clips, row));
        return;
    }
    if (lane == 0) blank_lp[row] = blank >= 0 && blank < V ? __ldg(x + blank) : -INFINITY;
    // K rounds of a warp arg-best; only the lane whose best was taken scans its columns again
    float pv = 0.0f;
    int pi = -1;   // the previous pick (none yet)
    auto scan = [&](float &bv, int &bi) {
        bi = -1;
        for (int v = lane; v < V; v += 32) {
            if (v == blank) continue;
            const float f = __ldg(x + v);
            if (pi >= 0 && !ranks_before(pv, pi, f, v)) continue;
            if (bi < 0 || ranks_before(f, v, bv, bi)) {
                bv = f;
                bi = v;
            }
        }
    };
    float bv = 0.0f;
    int bi;
    scan(bv, bi);
    for (int r = 0; r < K; ++r) {
        float wv = bv;
        int wi = bi;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(kFull, wv, o);
            const int oi = __shfl_xor_sync(kFull, wi, o);
            if (oi >= 0 && (wi < 0 || ranks_before(ov, oi, wv, wi))) {
                wv = ov;
                wi = oi;
            }
        }
        if (lane == 0) {
            top_id[row * K + r] = wi;
            top_lp[row * K + r] = wv;
        }
        pv = wv;
        pi = wi;
        if (bi == wi) scan(bv, bi);
    }
}

struct Smem {
    unsigned long long *keys, *surv, *order;
    Beam *cur, *nxt;
    Prelude *pre;
    float *keep_pb, *keep_pnb;
    int *top_id;
    float *top_lp;
    int *tab_node, *tab_beam;
    unsigned *hist;
    int *scalars;   // nb, survivors, merged, need; prefix in keys' tail
};

__host__ __device__ size_t align16(size_t x) { return (x + 15) & ~size_t(15); }

// The dynamic shared memory of beam_kernel for B beams and K candidate tokens: the bytes of each array, in order
constexpr int kSmemArrays = 14;
__host__ __device__ void smem_sizes(int B, int K, size_t *bytes) {
    const size_t b = (size_t)(B > 0 ? B : 1), sizes[kSmemArrays] = {
        b * (K + 1) * sizeof(unsigned long long),   // keys
        b * sizeof(unsigned long long),             // survivors
        b * sizeof(unsigned long long),             // their order
        b * sizeof(Beam),                           // cur
        b * sizeof(Beam),                           // nxt
        b * sizeof(Prelude),
        b * sizeof(float),                          // keep pb
        b * sizeof(float),                          // keep pnb
        (size_t)K * sizeof(int),
        (size_t)K * sizeof(float),
        (size_t)kTable * sizeof(int),
        (size_t)kTable * sizeof(int),
        (size_t)256 * sizeof(unsigned),
        (size_t)8 * sizeof(int) + sizeof(unsigned long long)};
    for (int i = 0; i < kSmemArrays; ++i) bytes[i] = align16(sizes[i]);
}

size_t beam_smem(int B, int K) {
    size_t bytes[kSmemArrays], n = 0;
    smem_sizes(B, K, bytes);
    for (size_t x : bytes) n += x;
    return n;
}

__device__ unsigned long long cas64(unsigned long long *p, unsigned long long expected, unsigned long long desired) {
    return atomicCAS(p, expected, desired);
}

__global__ void __launch_bounds__(kThreads, 1) beam_kernel(const ClipDesc *__restrict__ clips,
                                                          const int *__restrict__ top_id,
                                                          const float *__restrict__ top_lp,
                                                          const float *__restrict__ blank_lp, int B, int K,
                                                          const LmView *__restrict__ lm, float weight, float bonus,
                                                          Pieces pieces, unsigned long long *__restrict__ trie,
                                                          int *__restrict__ staged, long long *__restrict__ len_out,
                                                          float *__restrict__ score_out, const int *__restrict__ bad) {
    if (*bad != kNoBad) return;   // a refused call: the host reads nothing
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem S;
    {
        size_t bytes[kSmemArrays];
        smem_sizes(B, K, bytes);
        unsigned char *p[kSmemArrays];
        p[0] = smem_raw;
        for (int i = 1; i < kSmemArrays; ++i) p[i] = p[i - 1] + bytes[i - 1];
        S.keys = (unsigned long long *)p[0];
        S.surv = (unsigned long long *)p[1];
        S.order = (unsigned long long *)p[2];
        S.cur = (Beam *)p[3];
        S.nxt = (Beam *)p[4];
        S.pre = (Prelude *)p[5];
        S.keep_pb = (float *)p[6];
        S.keep_pnb = (float *)p[7];
        S.top_id = (int *)p[8];
        S.top_lp = (float *)p[9];
        S.tab_node = (int *)p[10];
        S.tab_beam = (int *)p[11];
        S.hist = (unsigned *)p[12];
        S.scalars = (int *)p[13];
    }
    unsigned long long *s_prefix = (unsigned long long *)(S.scalars + 8);
    const int tid = threadIdx.x;
    const ClipDesc clip = clips[blockIdx.x];
    unsigned long long *keys_trie = trie + clip.node0;
    const long long cap = clip.cap;
    for (long long s = tid; s < cap; s += kThreads) keys_trie[s] = kEmpty;
    if (tid == 0) {
        S.cur[0] = Beam{0.0f, -INFINITY, 0.0f, kRootNode, -1, kNoToken, 0, kLmRoot, kNoWord};
        S.scalars[0] = 1;
    }
    __syncthreads();
    const int KK = K + 1;
    auto cas = [&](long long s, unsigned long long e, unsigned long long d) { return cas64(keys_trie + s, e, d); };
    for (int t = 0; t < clip.frames; ++t) {
        const long long row = clip.row0 + t;
        const int nb = S.scalars[0];
        if (nb == 0) break;
        if (tid < K) {
            S.top_id[tid] = top_id[row * K + tid];
            S.top_lp[tid] = top_lp[row * K + tid];
        }
        for (int s = tid; s < kTable; s += kThreads) S.tab_node[s] = -1;
        if (tid == 0) S.scalars[2] = 0;
        __syncthreads();
        const float blank = blank_lp[row];
        for (int i = tid; i < nb; i += kThreads) {
            const Beam b = S.cur[i];
            S.pre[i] = prelude(b, lm, weight, bonus);
            for (unsigned h = (unsigned)mix((unsigned)b.node) & (kTable - 1);; h = (h + 1) & (kTable - 1)) {
                if (atomicCAS(&S.tab_node[h], -1, b.node) == -1) {
                    S.tab_beam[h] = i;
                    break;
                }
            }
        }
        __syncthreads();
        const int n = nb * KK;
        for (int s = tid; s < n; s += kThreads) {
            const int i = s / KK, c = s - i * KK;
            if (c == 0) continue;
            const int v = S.top_id[c - 1];
            const Beam &b = S.cur[i];
            const Prelude &p = S.pre[i];
            const float pnb = ext_pnb(b, p, v, S.top_lp[c - 1]);
            S.keys[s] = order_key(beam_total(-INFINITY, pnb, ext_lm(b, p, pieces.boundary[v] != 0)), s, s);
        }
        __syncthreads();
        for (int i = tid; i < nb; i += kThreads) {
            const Beam b = S.cur[i];
            int rc = -1;
            for (int c = 0; c < K && b.last >= 0; ++c)
                if (S.top_id[c] == b.last) rc = c;
            float pb, pnb;
            keep_start(b, S.pre[i], blank, rc >= 0, rc >= 0 ? S.top_lp[rc] : 0.0f, pb, pnb);
            int gen = i * KK;
            if (rc >= 0 && b.parent >= 0) {
                int j = -1;
                for (unsigned h = (unsigned)mix((unsigned)b.parent) & (kTable - 1);; h = (h + 1) & (kTable - 1)) {
                    const int x = S.tab_node[h];
                    if (x == b.parent) j = S.tab_beam[h];
                    if (x == b.parent || x == -1) break;
                }
                if (j >= 0) {   // the parent's extension by the last token is this prefix: folded in, its slot dead
                    pnb = log_add_exp(pnb, ext_pnb(S.cur[j], S.pre[j], b.last, S.top_lp[rc]));
                    const int slot = j * KK + 1 + rc;
                    gen = min(gen, slot);
                    S.keys[slot] = kEmpty;
                    atomicAdd(&S.scalars[2], 1);
                }
            }
            S.keep_pb[i] = pb;
            S.keep_pnb[i] = pnb;
            S.keys[i * KK] = order_key(beam_total(pb, pnb, b.lm), gen, i * KK);
        }
        __syncthreads();
        const int valid = n - S.scalars[2];
        const int keep = min(B, valid);
        // keep == 0 (beam_width 0) leaves no survivor and skips the select, whose digit search needs need >= 1
        unsigned long long thr = kEmpty - 1;
        if (keep > 0 && keep < valid) {   // radix select of the keep-th smallest key, 8 bits at a time from the top
            unsigned long long prefix = 0;
            int need = keep;
            for (int shift = 56; shift >= 0; shift -= 8) {
                for (int s = tid; s < 256; s += kThreads) S.hist[s] = 0;
                __syncthreads();
                const unsigned long long hi = shift == 56 ? 0ull : ~0ull << (shift + 8);
                for (int s = tid; s < n; s += kThreads) {
                    const unsigned long long k = S.keys[s];
                    if (k != kEmpty && (k & hi) == prefix) atomicAdd(&S.hist[(k >> shift) & 255], 1u);
                }
                __syncthreads();
                if (tid < 32) {
                    unsigned h[8], sum = 0;
#pragma unroll
                    for (int d = 0; d < 8; ++d) sum += (h[d] = S.hist[tid * 8 + d]);
                    unsigned incl = sum;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned y = __shfl_up_sync(kFull, incl, o);
                        if (tid >= o) incl += y;
                    }
                    unsigned cum = incl - sum;
                    if (cum < (unsigned)need && (unsigned)need <= incl) {
                        for (int d = 0; d < 8; ++d) {
                            if (cum + h[d] >= (unsigned)need) {
                                *s_prefix = prefix | ((unsigned long long)(tid * 8 + d) << shift);
                                S.scalars[3] = need - (int)cum;
                                break;
                            }
                            cum += h[d];
                        }
                    }
                }
                __syncthreads();
                prefix = *s_prefix;
                need = S.scalars[3];
            }
            thr = prefix;
        }
        if (tid == 0) S.scalars[1] = 0;
        __syncthreads();
        for (int s = tid; s < n; s += kThreads) {
            const unsigned long long k = S.keys[s];
            if (keep > 0 && k != kEmpty && k <= thr) S.surv[atomicAdd(&S.scalars[1], 1)] = k;
        }
        __syncthreads();
        const int ns = S.scalars[1];
        for (int r = tid; r < ns; r += kThreads) {
            const unsigned long long k = S.surv[r];
            int rank = 0;
            for (int q = 0; q < ns; ++q) rank += S.surv[q] < k;
            S.order[rank] = k;
        }
        __syncthreads();
        for (int r = tid; r < ns; r += kThreads) {
            const int slot = key_slot(S.order[r]);
            const int i = slot / KK, c = slot - i * KK;
            Beam nb_;
            if (c == 0) {
                nb_ = S.cur[i];
                nb_.pb = S.keep_pb[i];
                nb_.pnb = S.keep_pnb[i];
            } else {
                const Beam b = S.cur[i];
                const int v = S.top_id[c - 1];
                nb_ = ext_beam(b, S.pre[i], v, ext_pnb(b, S.pre[i], v, S.top_lp[c - 1]), lm, pieces);
                nb_.node = cons(keys_trie, cap, b.node, v, cas);
            }
            S.nxt[r] = nb_;
        }
        __syncthreads();
        Beam *tmp = S.cur;
        S.cur = S.nxt;
        S.nxt = tmp;
        if (tid == 0) S.scalars[0] = ns;
        __syncthreads();
    }
    const int nb = S.scalars[0];
    for (int i = tid; i < nb; i += kThreads) S.keep_pb[i] = final_total(S.cur[i], lm, weight, bonus);
    __syncthreads();
    if (tid == 0) {
        int best = 0;
        for (int i = 1; i < nb; ++i)
            if (S.keep_pb[i] > S.keep_pb[best]) best = i;
        if (nb == 0) {
            len_out[blockIdx.x] = 0;
            score_out[blockIdx.x] = -INFINITY;
        } else {
            const Beam b = S.cur[best];
            len_out[blockIdx.x] = b.len;
            score_out[blockIdx.x] = S.keep_pb[best];
            int node = b.node;
            for (int k = b.len - 1; k >= 0; --k) {
                staged[clip.row0 + k] = node_token(keys_trie, node);
                node = node_parent(keys_trie, node);
            }
        }
    }
}

__global__ void __launch_bounds__(kWarps * 32) argmax_kernel(const float *__restrict__ lp, long long rows, int V,
                                                              int *__restrict__ ids) {
    const long long row = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float *x = lp + row * V;
    float bv = -INFINITY;
    int bi = INT_MAX;   // no column of this lane yet
    for (int v = lane; v < V; v += 32) {
        const float f = __ldg(x + v);
        if (!isnan(f) && (bi == INT_MAX || f > bv)) {
            bv = f;
            bi = v;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(kFull, bv, o);
        const int oi = __shfl_xor_sync(kFull, bi, o);
        if (oi != INT_MAX && (bi == INT_MAX || greedy_better(ov, oi, bv, bi))) {
            bv = ov;
            bi = oi;
        }
    }
    if (lane == 0) ids[row] = bi == INT_MAX || isnan(__ldg(x)) ? 0 : bi;
}

__global__ void __launch_bounds__(kThreads) collapse_kernel(const ClipDesc *__restrict__ clips,
                                                              const int *__restrict__ ids, int blank,
                                                              int *__restrict__ staged, long long *__restrict__ len) {
    __shared__ int warp_sum[kThreads / 32];
    const ClipDesc clip = clips[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int *id = ids + clip.row0;
    int base = 0;
    for (int start = 0; start < clip.frames; start += kThreads) {
        const int t = start + tid;
        const bool keep = t < clip.frames && greedy_keep(id[t], t > 0 ? id[t - 1] : kNoToken, blank);
        const unsigned ballot = __ballot_sync(kFull, keep);
        if (lane == 0) warp_sum[w] = __popc(ballot);
        __syncthreads();
        int before = __popc(ballot & ((1u << lane) - 1)), all = 0;
        for (int q = 0; q < kThreads / 32; ++q) {
            before += q < w ? warp_sum[q] : 0;
            all += warp_sum[q];
        }
        if (keep) staged[clip.row0 + base + before] = id[t];
        base += all;
        __syncthreads();
    }
    if (tid == 0) len[blockIdx.x] = base;
}

__global__ void __launch_bounds__(kThreads) gather_kernel(const ClipDesc *__restrict__ clips,
                                                            const int *__restrict__ staged,
                                                            const long long *__restrict__ len,
                                                            const long long *__restrict__ offsets,
                                                            int32_t *__restrict__ out) {
    const ClipDesc clip = clips[blockIdx.x];
    const long long n = len[blockIdx.x], o = offsets[blockIdx.x];
    for (long long k = threadIdx.x; k < n; k += kThreads) out[o + k] = staged[clip.row0 + k];
}

unsigned blocks_for(long long n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

// The clip descriptors and the row offsets at the head of `stage`, uploaded; the output offsets go at `off_at` later
int stage_clips(UploadStage<> &stage, cudaStream_t stream, const int64_t *row_offsets, int clips, int B,
                size_t &off_at, long long &nodes) {
    std::vector<ClipDesc> cd((size_t)clips);
    nodes = 0;
    for (int b = 0; b < clips; ++b) {
        const long long T = row_offsets[b + 1] - row_offsets[b];
        const long long cap = 2 * T * B + 1;
        cd[(size_t)b] = ClipDesc{row_offsets[b], nodes, cap, (int)T, 0};
        nodes += cap;
    }
    const size_t clip_bytes = cd.size() * sizeof(ClipDesc), offs_bytes = ((size_t)clips + 1) * sizeof(long long);
    off_at = (clip_bytes + offs_bytes + 255) & ~size_t(255);
    const int st = stage.reserve(off_at + (size_t)clips * sizeof(long long));
    if (st != FA_OK) return st;
    char *h = static_cast<char *>(stage.host.data());
    std::memcpy(h, cd.data(), clip_bytes);
    std::memcpy(h + clip_bytes, row_offsets, offs_bytes);
    return stage.upload(clip_bytes + offs_bytes, stream);
}

// After the one synchronisation: lengths and the total, the output offsets uploaded behind them.  FA_OUTPUT_TOO_SMALL
// when the capacity is short.
int plan_output(UploadStage<> &stage, cudaStream_t stream, const long long *h_len, int clips, size_t off_at,
                int64_t *lengths, int64_t *total, long long capacity, const char *entry) {
    long long *off = reinterpret_cast<long long *>(static_cast<char *>(stage.host.data()) + off_at);
    long long sum = 0;
    for (int b = 0; b < clips; ++b) {
        off[b] = sum;
        lengths[b] = h_len[b];
        sum += h_len[b];
    }
    *total = sum;
    if (sum > capacity) {
        set_error("%s: %lld tokens, capacity %lld", entry, sum, capacity);
        return FA_OUTPUT_TOO_SMALL;
    }
    if (sum == 0) return FA_OK;
    FA_CUDA_TRY(cudaMemcpyAsync(static_cast<char *>(stage.device.data()) + off_at, off, (size_t)clips * sizeof(long long),
                                cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaEventRecord(stage.uploaded, stream));
    stage.in_flight = true;   // the next reserve() waits for this copy out of the pinned buffer
    return FA_OK;
}

int gather(UploadStage<> &stage, DeviceBuffer<> &d_buf, cudaStream_t stream, bool on_device, int clips, size_t off_at,
           const int *d_staged, const long long *d_len, long long total, int32_t *tokens) {
    HostStaging O(!on_device, stream);
    int32_t *d_tok;
    const int st = O.carve(d_buf, [&](HostStaging::Layout &l) { d_tok = l.out(tokens, (size_t)total); });
    if (st != FA_OK) return st;
    const char *d = static_cast<const char *>(stage.device.data());
    FA_CUDA_TRY(launch(gather_kernel, dim3((unsigned)clips), dim3(kThreads), 0, stream,
                       reinterpret_cast<const ClipDesc *>(d), d_staged, d_len,
                       reinterpret_cast<const long long *>(d + off_at), d_tok));
    FA_CUDA_TRY(O.finish());
    return FA_OK;
}

} // namespace

// ------------------------------------------------------------------------------------------------ host
int Lm::init(const LmTables &t) {
    FA_CUDA_TRY(cudaGetDevice(&device));
    int st = stream.create();
    if (st != FA_OK) return st;
    const unsigned long long *ck, *bk;
    const int *cn, *nw;
    const float *ulp, *ubo, *blp;
    LmView *dv;
    auto layout = [&](Carver &c) {
        dv = c.take<LmView>(1);
        ck = c.take<unsigned long long>(t.child_key.size());
        bk = c.take<unsigned long long>(t.bigram_key.size());
        cn = c.take<int>(t.child_node.size());
        nw = c.take<int>(t.node_word.size());
        ulp = c.take<float>(t.uni_log_prob.size() + 1);
        ubo = c.take<float>(t.uni_backoff.size() + 1);
        blp = c.take<float>(t.bigram_log_prob.size());
    };
    st = carve_arena(d, layout);
    if (st != FA_OK) return st;
    auto put = [&](const void *dst, const auto &v) {
        return v.empty() ? cudaSuccess
                         : cudaMemcpyAsync(const_cast<void *>(dst), v.data(), v.size() * sizeof(v[0]),
                                           cudaMemcpyHostToDevice, stream);
    };
    FA_CUDA_TRY(put(ck, t.child_key));
    FA_CUDA_TRY(put(bk, t.bigram_key));
    FA_CUDA_TRY(put(cn, t.child_node));
    FA_CUDA_TRY(put(nw, t.node_word));
    FA_CUDA_TRY(put(ulp, t.uni_log_prob));
    FA_CUDA_TRY(put(ubo, t.uni_backoff));
    FA_CUDA_TRY(put(blp, t.bigram_log_prob));
    view = LmView{ck, cn, (long long)t.child_key.size(), nw, ulp, ubo, bk, blp, (long long)t.bigram_key.size()};
    FA_CUDA_TRY(cudaMemcpyAsync(dv, &view, sizeof(view), cudaMemcpyHostToDevice, stream));
    // complete before fa_ctc_lm_create returns: a decoder's stream is not ordered after this one
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    d_view = dv;
    return FA_OK;
}

int Decoder::init(int vocab_, int blank_, const char *bytes, const int64_t *offsets) {
    vocab = vocab_;
    blank_id = blank_;
    FA_CUDA_TRY(cudaGetDevice(&device));
    int st = stream.create();
    if (st != FA_OK) return st;
    const long long n_bytes = offsets[vocab];
    std::vector<unsigned char> boundary((size_t)vocab);
    for (int v = 0; v < vocab; ++v) {
        const unsigned char *p = reinterpret_cast<const unsigned char *>(bytes) + offsets[v];
        boundary[(size_t)v] = offsets[v + 1] - offsets[v] >= 3 && p[0] == 0xE2 && p[1] == 0x96 && p[2] == 0x81;
    }
    long long *d_off;
    unsigned char *d_bound, *d_bytes;
    st = carve_arena(d_pieces, [&](Carver &c) {
        d_off = c.take<long long>((size_t)vocab + 1);
        d_bound = c.take<unsigned char>((size_t)vocab);
        d_bytes = c.take<unsigned char>((size_t)n_bytes + 1);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(cudaMemcpyAsync(d_off, offsets, ((size_t)vocab + 1) * sizeof(long long), cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(d_bound, boundary.data(), (size_t)vocab, cudaMemcpyHostToDevice, stream));
    if (n_bytes) FA_CUDA_TRY(cudaMemcpyAsync(d_bytes, bytes, (size_t)n_bytes, cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    pieces = Pieces{d_bytes, d_off, d_bound};
    return FA_OK;
}

int Decoder::beam_search(const Lm *lm, bool on_device, const float *log_probs, const int64_t *row_offsets, int clips,
                         int B, int K, float weight, float bonus, int64_t *lengths, float *scores, int32_t *tokens,
                         long long capacity, int64_t *total) {
    FA_CUDA_TRY(cudaSetDevice(device));
    if (clips == 0) {
        *total = 0;
        return FA_OK;
    }
    const long long rows = row_offsets[clips];
    size_t off_at;
    long long nodes;
    int st = stage_clips(stage, stream, row_offsets, clips, B, off_at, nodes);
    if (st != FA_OK) return st;
    const char *d = static_cast<const char *>(stage.device.data());
    const auto *d_clips = reinterpret_cast<const ClipDesc *>(d);
    const auto *d_offs = reinterpret_cast<const long long *>(d + (size_t)clips * sizeof(ClipDesc));
    int *d_top_id, *d_staged, *d_bad;
    float *d_top_lp, *d_blank, *d_score;
    unsigned long long *d_trie;
    long long *d_len;
    st = carve_arena(scratch, [&](Carver &c) {
        d_top_id = c.take<int>((size_t)rows * K);
        d_top_lp = c.take<float>((size_t)rows * K);
        d_blank = c.take<float>((size_t)rows);
        d_trie = c.take<unsigned long long>((size_t)nodes);
        d_staged = c.take<int>((size_t)rows);
        d_len = c.take<long long>((size_t)clips);
        d_score = c.take<float>((size_t)clips);
        d_bad = c.take<int>(1);
    });
    if (st != FA_OK) return st;
    const size_t res_bytes = (size_t)clips * (sizeof(long long) + sizeof(float)) + sizeof(int);
    st = h_res.grow(res_bytes);
    if (st != FA_OK) return st;
    HostStaging H(!on_device, stream);
    const float *d_lp;
    st = H.carve(d_buf, [&](HostStaging::Layout &l) { d_lp = l.in(log_probs, (size_t)rows * vocab); });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(cudaMemsetAsync(d_bad, 0x7f, sizeof(int), stream));
    if (rows > 0)
        FA_CUDA_TRY(launch(topk_kernel, dim3(blocks_for(rows, kWarps)), dim3(kWarps * 32), 0, stream, d_lp, rows, vocab,
                           blank_id, K, d_offs, clips, d_top_id, d_top_lp, d_blank, d_bad));
    const size_t smem = beam_smem(B, K);
    FA_CUDA_TRY(cudaFuncSetAttribute(beam_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FA_CUDA_TRY(launch(beam_kernel, dim3((unsigned)clips), dim3(kThreads), smem, stream, d_clips, d_top_id, d_top_lp,
                       d_blank, B, K, lm ? lm->d_view : nullptr, weight, bonus, pieces, d_trie, d_staged,
                       d_len, d_score, d_bad));
    char *h = static_cast<char *>(h_res.data());
    auto *h_len = reinterpret_cast<long long *>(h);
    auto *h_score = reinterpret_cast<float *>(h + (size_t)clips * sizeof(long long));
    auto *h_bad = reinterpret_cast<int *>(h + (size_t)clips * (sizeof(long long) + sizeof(float)));
    FA_CUDA_TRY(cudaMemcpyAsync(h_len, d_len, (size_t)clips * sizeof(long long), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(h_score, d_score, (size_t)clips * sizeof(float), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(h_bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    if (*h_bad != kNoBad) {
        set_error("fa_ctc_beam_search: clip %d has a NaN or +inf log-prob", *h_bad);
        return FA_INVALID_ARGUMENT;
    }
    for (int b = 0; b < clips; ++b) scores[b] = h_score[b];
    st = plan_output(stage, stream, h_len, clips, off_at, lengths, total, capacity, "fa_ctc_beam_search");
    if (st != FA_OK || *total == 0) return st;
    return gather(stage, d_buf, stream, on_device, clips, off_at, d_staged, d_len, *total, tokens);
}

int greedy(CallContext &C, bool on_device, const float *log_probs, const int64_t *row_offsets, int clips, int vocab,
           int blank_id, int64_t *lengths, int32_t *tokens, long long capacity, int64_t *total) {
    *total = 0;
    if (clips == 0) return FA_OK;
    const long long rows = row_offsets[clips];
    size_t off_at;
    long long nodes;
    int st = stage_clips(C.stage, C.stream, row_offsets, clips, 0, off_at, nodes);
    if (st != FA_OK) return st;
    const auto *d_clips = static_cast<const ClipDesc *>(C.stage.device.data());
    int *d_ids, *d_staged;
    long long *d_len;
    st = carve_arena(C.scratch, [&](Carver &c) {
        d_ids = c.take<int>((size_t)rows);
        d_staged = c.take<int>((size_t)rows);
        d_len = c.take<long long>((size_t)clips);
    });
    if (st != FA_OK) return st;
    st = C.h_buf.grow((size_t)clips * sizeof(long long));
    if (st != FA_OK) return st;
    HostStaging H(!on_device, C.stream);
    const float *d_lp;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) { d_lp = l.in(log_probs, (size_t)rows * vocab); });
    if (st != FA_OK) return st;
    if (rows > 0)
        FA_CUDA_TRY(launch(argmax_kernel, dim3(blocks_for(rows, kWarps)), dim3(kWarps * 32), 0, C.stream, d_lp, rows,
                           vocab, d_ids));
    FA_CUDA_TRY(launch(collapse_kernel, dim3((unsigned)clips), dim3(kThreads), 0, C.stream, d_clips, d_ids, blank_id,
                       d_staged, d_len));
    auto *h_len = static_cast<long long *>(C.h_buf.data());
    FA_CUDA_TRY(cudaMemcpyAsync(h_len, d_len, (size_t)clips * sizeof(long long), cudaMemcpyDeviceToHost, C.stream));
    FA_CUDA_TRY(cudaStreamSynchronize(C.stream));
    st = plan_output(C.stage, C.stream, h_len, clips, off_at, lengths, total, capacity, "fa_ctc_greedy");
    if (st != FA_OK || *total == 0) return st;
    return gather(C.stage, C.d_buf, C.stream, on_device, clips, off_at, d_staged, d_len, *total, tokens);
}

} // namespace ctc_decode
} // namespace fa
