// CTC keyword spotting on the GPU (ctc_core.cuh holds the arithmetic):
//
//   log_softmax_kernel   one thread per row: applyLogSoftmax, the exp sum in index order
//   merge_chunks_kernel  one thread per output element: the row's sources folded with mergeOverlapFrame in chunk order
//   spot_kernel          one warp per (clip, term) pair: the CTC-WS dynamic program over the clip, each lane holding 8
//                        consecutive expanded states in registers (s - 1 and s - 2 of its first states come from the
//                        lane below by shuffle), the candidate scan one frame behind, then lane 0 sorts and merges
//                        the pair's candidates in its scratch slots and writes the pair's count
//   compact_kernel       one warp per pair: its merged detections to their place in the output
//   constrained_kernel   one warp per query: the same dynamic program over the query's window
//
// No parallelism in time: the pairs (and queries) are independent, and each walks its frames in order.
#include "ctc_spot.h"

#include "ctc_core.cuh"

#include <algorithm>
#include <climits>
#include <cstring>

namespace fa {
namespace ctc {

namespace {

constexpr int kRowThreads = 128;
constexpr int kWarps = 4;   // pairs per CTA of spot_kernel / queries per CTA of constrained_kernel
constexpr unsigned kFull = 0xffffffffu;

__global__ void __launch_bounds__(kRowThreads) log_softmax_kernel(const float *__restrict__ x, int frames, int V,
                                                                   int layout, float temperature, float bias,
                                                                   int blank, float *__restrict__ out) {
    const long long t = (long long)blockIdx.x * kRowThreads + threadIdx.x;
    if (t >= frames) return;
    const long long step = layout == kVocabMajor ? frames : 1;
    const float *src = x + (layout == kVocabMajor ? t : t * V);
    float *dst = out + t * V;
    log_softmax_row(V, temperature, bias, blank, [&](int v) { return __ldg(src + v * step); },
                    [&](int v, float r) { dst[v] = r; });
}

__global__ void __launch_bounds__(kRowThreads) merge_chunks_kernel(const float *__restrict__ in, int V,
                                                                    long long out_rows,
                                                                    const long long *__restrict__ row_src,
                                                                    const long long *__restrict__ src,
                                                                    float *__restrict__ out) {
    const long long n = out_rows * V;
    for (long long i = (long long)blockIdx.x * kRowThreads + threadIdx.x; i < n;
         i += (long long)gridDim.x * kRowThreads) {
        const long long r = i / V, v = i - r * V;
        long long k = row_src[r];
        const long long end = row_src[r + 1];
        float a = in[src[k] * V + v];
        for (++k; k < end; ++k) a = merge_overlap(a, in[src[k] * V + v]);
        out[i] = a;
    }
}

// The warp's dynamic program over `frames` rows of lp, calling on_frame(t, dp[t][N] cell) for t = 1 .. frames (every
// lane, with the same values).  tok(i) reads the term's token i; n_tokens >= 1 and 2N + 1 <= kMaxStates.
template <typename Tok, typename OnFrame>
__device__ __forceinline__ void warp_dp(const float *__restrict__ lp, int frames, int V, int blank, Tok tok,
                                        int n_tokens, OnFrame &&on_frame) {
    const int lane = threadIdx.x & 31;
    const int n_states = 2 * n_tokens + 1;
    State st[kStatesPerLane];
    Cell c[kStatesPerLane];
#pragma unroll
    for (int j = 0; j < kStatesPerLane; ++j) {
        const int s = lane * kStatesPerLane + j;
        st[j] = s < n_states ? expanded_state(s, tok, V, blank) : State{kEmitZero, false, false};
        c[j] = Cell{s == 0 ? 0.0f : kNeg, 0, 0};
    }
    const int s_tok = 2 * n_tokens - 1, s_blank = 2 * n_tokens;
    const int tok_lane = s_tok / kStatesPerLane, tok_j = s_tok % kStatesPerLane;
    const int blank_lane = s_blank / kStatesPerLane, blank_j = s_blank % kStatesPerLane;
    float e[kStatesPerLane];
#pragma unroll
    for (int j = 0; j < kStatesPerLane; ++j) e[j] = frames > 0 ? emission(st[j], lp) : 0.0f;
    for (int t = 1; t <= frames; ++t) {
        float en[kStatesPerLane];   // the next frame's emissions, loaded while this frame is computed
        const float *next = lp + (long long)t * V;
#pragma unroll
        for (int j = 0; j < kStatesPerLane; ++j) en[j] = t < frames ? emission(st[j], next) : 0.0f;
        Cell p7, p6;   // states s - 1 and s - 2 of this lane's first state, at t - 1
        p7.dp = __shfl_up_sync(kFull, c[7].dp, 1);
        p7.start = __shfl_up_sync(kFull, c[7].start, 1);
        p7.last = __shfl_up_sync(kFull, c[7].last, 1);
        p6.dp = __shfl_up_sync(kFull, c[6].dp, 1);
        p6.start = __shfl_up_sync(kFull, c[6].start, 1);
        p6.last = __shfl_up_sync(kFull, c[6].last, 1);
#pragma unroll
        for (int j = kStatesPerLane - 1; j >= 0; --j) {
            const int s = lane * kStatesPerLane + j;
            if (s == 0) {
                c[0] = Cell{0.0f, t, 0};
            } else if (s < n_states) {
                const Cell adv = j >= 1 ? c[j - 1] : p7;
                const Cell skip = j >= 2 ? c[j - 2] : (j == 1 ? p7 : p6);
                c[j] = step_cell(c[j], adv, skip, st[j], e[j], t, s);
            }
        }
        Cell mine_tok = c[0], mine_blank = c[0];
#pragma unroll
        for (int j = 1; j < kStatesPerLane; ++j) {
            if (j == tok_j) mine_tok = c[j];
            if (j == blank_j) mine_blank = c[j];
        }
        Cell a, b;
        a.dp = __shfl_sync(kFull, mine_tok.dp, tok_lane);
        a.start = __shfl_sync(kFull, mine_tok.start, tok_lane);
        a.last = __shfl_sync(kFull, mine_tok.last, tok_lane);
        b.dp = __shfl_sync(kFull, mine_blank.dp, blank_lane);
        b.start = __shfl_sync(kFull, mine_blank.start, blank_lane);
        b.last = __shfl_sync(kFull, mine_blank.last, blank_lane);
        on_frame(t, project(a, b));
#pragma unroll
        for (int j = 0; j < kStatesPerLane; ++j) e[j] = en[j];
    }
}

__global__ void __launch_bounds__(kWarps * 32) spot_kernel(const float *__restrict__ lp, int V, int blank,
                                                             const ClipDesc *__restrict__ clips, int K,
                                                             const TermDesc *__restrict__ terms,
                                                             const int *__restrict__ tokens,
                                                             const float *__restrict__ thresholds,
                                                             Candidate *__restrict__ cand, int *__restrict__ counts) {
    const int per_clip = (K + kWarps - 1) / kWarps;   // CTAs of one clip
    const int b = blockIdx.x / per_clip, k = (blockIdx.x % per_clip) * kWarps + (threadIdx.x >> 5);
    if (k >= K) return;
    const int lane = threadIdx.x & 31;
    const ClipDesc clip = clips[b];
    const TermDesc term = terms[k];
    const long long pair = (long long)b * K + k;
    if (term.count == 0 || clip.frames < term.count) {   // N == 0, T == 0 and T < N give nothing
        if (lane == 0) counts[pair] = 0;
        return;
    }
    Candidate *mine = cand + clip.cand0 + (long long)k * clip.cap;
    const int *tk = tokens + term.offset;
    const int N = term.count;
    Scan scan;
    scan.init(term.norm, thresholds[k]);
    int n = 0;
    auto emit = [&](const Candidate &x) {
        if (lane == 0) mine[n] = x;
        ++n;
    };
    warp_dp(lp + clip.row0 * V, clip.frames, V, blank, [&](int i) { return __ldg(tk + i); }, N,
            [&](int t, const Cell &cell) {
                if (t >= N) scan.push(cell, emit);
            });
    scan.finish(emit);
    if (lane == 0) counts[pair] = merge_candidates(mine, n);
}

__global__ void __launch_bounds__(kWarps * 32) compact_kernel(int B, int K, const ClipDesc *__restrict__ clips,
                                                                const Candidate *__restrict__ cand,
                                                                const int *__restrict__ counts,
                                                                const long long *__restrict__ offsets,
                                                                fa_ctc_detection *__restrict__ out) {
    const long long pair = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (pair >= (long long)B * K) return;
    const int b = (int)(pair / K), k = (int)(pair - (long long)b * K);
    const ClipDesc clip = clips[b];
    const Candidate *mine = cand + clip.cand0 + (long long)k * clip.cap;
    fa_ctc_detection *dst = out + offsets[pair];
    for (int i = threadIdx.x & 31; i < counts[pair]; i += 32) {
        const Candidate x = mine[i];
        dst[i] = fa_ctc_detection{b, k, x.score, x.start, x.end};
    }
}

__global__ void __launch_bounds__(kWarps * 32) constrained_kernel(const float *__restrict__ lp, int V, int blank,
                                                                    int Q, const QueryDesc *__restrict__ queries,
                                                                    const int *__restrict__ tokens,
                                                                    float *__restrict__ score,
                                                                    int64_t *__restrict__ start_frame,
                                                                    int64_t *__restrict__ end_frame) {
    const int q = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (q >= Q) return;
    const bool lead = (threadIdx.x & 31) == 0;
    const QueryDesc d = queries[q];
    const int N = d.count;
    if (N == 0 || d.frames < N) {   // empty query, empty window or a window shorter than the query
        if (lead) {
            score[q] = -INFINITY;
            start_frame[q] = end_frame[q] = d.start;
        }
        return;
    }
    const int *tk = tokens + d.offset;
    Cell best{kNeg, 0, 0};
    warp_dp(lp + d.start * V, (int)d.frames, V, blank, [&](int i) { return __ldg(tk + i); }, N,
            [&](int t, const Cell &cell) {
                if (t >= N && cell.dp > best.dp) best = cell;
            });
    if (lead) {
        const int norm = non_wildcard_count([&](int i) { return __ldg(tk + i); }, N);
        score[q] = norm > 0 ? fp::f_div(best.dp, (float)norm) : best.dp;
        start_frame[q] = d.start + best.start;
        end_frame[q] = d.start + best.last;
    }
}

unsigned blocks_for(long long n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

} // namespace

// ------------------------------------------------------------------------------------------------ host
int log_softmax(CallContext &C, bool on_device, const float *logits, int frames, int vocab, int layout,
                float temperature, float blank_bias, int blank_id, float *log_probs) {
    const size_t n = (size_t)frames * vocab;
    HostStaging H(!on_device, C.stream);
    const float *d_in;
    float *d_out;
    const int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_in = l.in(logits, n);
        d_out = l.out(log_probs, n);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(log_softmax_kernel, dim3(blocks_for(frames, kRowThreads)), dim3(kRowThreads), 0, C.stream,
                       d_in, frames, vocab, layout, temperature, blank_bias, blank_id, d_out));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int merge_chunks(CallContext &C, bool on_device, const float *chunks, long long in_rows, int vocab,
                 const std::vector<long long> &row_src, const std::vector<long long> &src, float *out) {
    const long long out_rows = (long long)row_src.size() - 1;
    const size_t desc_bytes = (row_src.size() + src.size()) * sizeof(long long);
    int st = C.stage.reserve(desc_bytes);
    if (st != FA_OK) return st;
    auto *h = static_cast<long long *>(C.stage.host.data());
    std::memcpy(h, row_src.data(), row_src.size() * sizeof(long long));
    std::memcpy(h + row_src.size(), src.data(), src.size() * sizeof(long long));
    st = C.stage.upload(desc_bytes, C.stream);
    if (st != FA_OK) return st;
    const auto *d_desc = static_cast<const long long *>(C.stage.device.data());
    HostStaging H(!on_device, C.stream);
    const float *d_in;
    float *d_out;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_in = l.in(chunks, (size_t)in_rows * vocab);
        d_out = l.out(out, (size_t)out_rows * vocab);
    });
    if (st != FA_OK) return st;
    const long long n = out_rows * vocab;
    const unsigned grid = (unsigned)std::min<long long>(blocks_for(n, kRowThreads), 132LL * 16);
    FA_CUDA_TRY(launch(merge_chunks_kernel, dim3(grid), dim3(kRowThreads), 0, C.stream, d_in, vocab, out_rows, d_desc,
                       d_desc + row_src.size(), d_out));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int spot_constrained(CallContext &C, bool on_device, const float *log_probs, int frames, int vocab, int blank_id,
                     const std::vector<QueryDesc> &queries, const std::vector<int> &tokens, float *score,
                     int64_t *start_frame, int64_t *end_frame) {
    const int Q = (int)queries.size();
    const size_t q_bytes = queries.size() * sizeof(QueryDesc), tok_bytes = tokens.size() * sizeof(int);
    int st = C.stage.reserve(q_bytes + tok_bytes);
    if (st != FA_OK) return st;
    char *h = static_cast<char *>(C.stage.host.data());
    std::memcpy(h, queries.data(), q_bytes);
    if (tok_bytes) std::memcpy(h + q_bytes, tokens.data(), tok_bytes);
    st = C.stage.upload(q_bytes + tok_bytes, C.stream);
    if (st != FA_OK) return st;
    const char *d = static_cast<const char *>(C.stage.device.data());
    HostStaging H(!on_device, C.stream);
    const float *d_lp;
    float *d_score;
    int64_t *d_start, *d_end;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_lp = l.in(log_probs, (size_t)frames * vocab);
        d_score = l.out(score, (size_t)Q);
        d_start = l.out(start_frame, (size_t)Q);
        d_end = l.out(end_frame, (size_t)Q);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(constrained_kernel, dim3(blocks_for(Q, kWarps)), dim3(kWarps * 32), 0, C.stream, d_lp, vocab,
                       blank_id, Q, reinterpret_cast<const QueryDesc *>(d),
                       reinterpret_cast<const int *>(d + q_bytes), d_score, d_start, d_end));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int Spotter::init(int vocab_, int blank_, int terms_, const int32_t *tokens, const int64_t *offsets) {
    vocab = vocab_;
    blank_id = blank_;
    terms = terms_;
    FA_CUDA_TRY(cudaGetDevice(&device));
    int st = stream.create();
    if (st != FA_OK) return st;
    const long long n_tok = terms ? offsets[terms] : 0;
    std::vector<TermDesc> desc((size_t)terms);
    term_len.resize((size_t)terms);
    for (int k = 0; k < terms; ++k) {
        const int off = (int)offsets[k], n = (int)(offsets[k + 1] - offsets[k]);
        const int nw = non_wildcard_count([&](int i) { return (int)tokens[off + i]; }, n);
        desc[(size_t)k] = TermDesc{off, n, nw > 0 ? (float)nw : 1.0f, 0};
        term_len[(size_t)k] = n;
    }
    const size_t desc_bytes = desc.size() * sizeof(TermDesc), tok_bytes = (size_t)n_tok * sizeof(int);
    st = d_terms.grow(desc_bytes + tok_bytes + 1);
    if (st != FA_OK) return st;
    char *d = static_cast<char *>(d_terms.data());
    // on the stream the kernels read them on, complete before `desc` and the caller's tokens go
    if (desc_bytes) FA_CUDA_TRY(cudaMemcpyAsync(d, desc.data(), desc_bytes, cudaMemcpyHostToDevice, stream));
    if (tok_bytes) FA_CUDA_TRY(cudaMemcpyAsync(d + desc_bytes, tokens, tok_bytes, cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    return FA_OK;
}

int Spotter::spot(bool on_device, const float *log_probs, const int64_t *row_offsets, int clips,
                  const float *min_score, int64_t *counts, int64_t *total, fa_ctc_detection *detections,
                  long long capacity) {
    FA_CUDA_TRY(cudaSetDevice(device));
    const long long pairs = (long long)clips * terms;
    *total = 0;
    for (long long p = 0; p < pairs; ++p) counts[p] = 0;
    if (pairs == 0) return FA_OK;
    // descriptors: clips, then thresholds, then (after the counts) each pair's first detection
    std::vector<ClipDesc> cd((size_t)clips);
    long long cand = 0;
    for (int b = 0; b < clips; ++b) {
        const int T = (int)(row_offsets[b + 1] - row_offsets[b]);
        cd[(size_t)b] = ClipDesc{row_offsets[b], cand, T, candidate_cap(T)};
        cand += (long long)terms * candidate_cap(T);
    }
    const size_t clip_bytes = cd.size() * sizeof(ClipDesc), thr_bytes = (size_t)terms * sizeof(float);
    const size_t off_at = (clip_bytes + thr_bytes + 255) & ~size_t(255), off_bytes = (size_t)pairs * sizeof(long long);
    int st = stage.reserve(off_at + off_bytes);
    if (st != FA_OK) return st;
    char *h = static_cast<char *>(stage.host.data());
    std::memcpy(h, cd.data(), clip_bytes);
    float *thr = reinterpret_cast<float *>(h + clip_bytes);
    for (int k = 0; k < terms; ++k) thr[k] = term_threshold(min_score != nullptr, min_score ? *min_score : 0.0f,
                                                            term_len[(size_t)k]);
    st = stage.upload(clip_bytes + thr_bytes, stream);
    if (st != FA_OK) return st;
    const char *d = static_cast<const char *>(stage.device.data());
    const auto *d_clips = reinterpret_cast<const ClipDesc *>(d);

    Candidate *d_cand = nullptr;
    int *d_counts = nullptr;
    st = carve_arena(scratch, [&](Carver &c) {
        d_cand = c.take<Candidate>((size_t)cand);
        d_counts = c.take<int>((size_t)pairs);
    });
    if (st != FA_OK) return st;
    st = h_counts.grow((size_t)pairs * sizeof(int));
    if (st != FA_OK) return st;
    HostStaging H(!on_device, stream);
    const float *d_lp;
    st = H.carve(d_buf, [&](HostStaging::Layout &l) { d_lp = l.in(log_probs, (size_t)row_offsets[clips] * vocab); });
    if (st != FA_OK) return st;
    const char *d_tok = static_cast<const char *>(d_terms.data()) + (size_t)terms * sizeof(TermDesc);
    FA_CUDA_TRY(launch(spot_kernel, dim3((unsigned)(blocks_for(terms, kWarps) * clips)), dim3(kWarps * 32), 0, stream,
                       d_lp, vocab, blank_id, d_clips, terms, static_cast<const TermDesc *>(d_terms.data()),
                       reinterpret_cast<const int *>(d_tok), reinterpret_cast<const float *>(d + clip_bytes), d_cand,
                       d_counts));
    FA_CUDA_TRY(cudaMemcpyAsync(h_counts.data(), d_counts, (size_t)pairs * sizeof(int), cudaMemcpyDeviceToHost, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    long long *off = reinterpret_cast<long long *>(h + off_at);
    long long sum = 0;
    for (long long p = 0; p < pairs; ++p) {
        off[p] = sum;
        counts[p] = h_counts.data()[p];
        sum += h_counts.data()[p];
    }
    *total = sum;
    if (sum > capacity) {
        set_error("fa_ctc_spot: %lld detections, capacity %lld", sum, capacity);
        return FA_OUTPUT_TOO_SMALL;
    }
    if (sum == 0) return FA_OK;
    FA_CUDA_TRY(cudaMemcpyAsync(static_cast<char *>(stage.device.data()) + off_at, off, off_bytes,
                                cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaEventRecord(stage.uploaded, stream));
    HostStaging O(!on_device, stream);
    fa_ctc_detection *d_det;
    // the log-probs' twin is no longer read: the detections' twin may take its place
    st = O.carve(d_buf, [&](HostStaging::Layout &l) { d_det = l.out(detections, (size_t)sum); });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(compact_kernel, dim3(blocks_for(pairs, kWarps)), dim3(kWarps * 32), 0, stream, clips, terms,
                       d_clips, d_cand, d_counts, reinterpret_cast<const long long *>(d + off_at), d_det));
    FA_CUDA_TRY(O.finish());
    return FA_OK;
}

} // namespace ctc
} // namespace fa
