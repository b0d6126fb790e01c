// Sortformer's streaming state update on the GPU (interface: sortformer_plan.h; arithmetic: sortformer_core.cuh).
//
//   sortformer_update_kernel   one CTA per session: fifoPreds overwrite, FIFO append, confirmed / tentative rows, the
//                              pop into the silence profile and the speaker cache, and compressSpkcache
//   sortformer_inputs_kernel   one CTA per (session, row): the next model call's spkcache / fifo tensors, zero padded
//
// An update push is one launch, a model-input gather one launch, whatever the session count.
//
// Compression runs in shared memory: the scores [L x 4] (L = the cache length after the pop), the speaker-major
// permuted values [(L + sil) x 4] with the +inf placeholders, one flag per permuted index and the kept frame of each
// output slot.  Both selections count ranks under `precedes` (sortformer_core.cuh): an element is kept when fewer than
// k elements precede it, which is the set the reference's insertion sorts keep, in the same order.  Rank counting was
// chosen over a bitonic sort because it needs no padding to a power of two, no tie-break payload and no extra pass for
// the per-speaker variants; at the sizes here (L*4 <= 2 300 values) its O(n^2) comparisons read shared memory as
// broadcasts.  The kept indices are sorted ascending by an exclusive prefix sum over the flags.
#include "sortformer_plan.h"

#include <algorithm>

namespace fa {
namespace sortformer {

namespace {

constexpr int kThreads = 256;
constexpr size_t kMaxDynamicSmem = 200 * 1024;

struct Smem {
    float *scores;   // [cache_rows x 4]
    float *perm;     // [(cache_rows + sil) x 4]
    int *flag;       // [(cache_rows + sil) x 4]
    int *slot;       // [spkcache_len]
    int *scan;       // [kThreads + 1]
    size_t bytes;
};

__host__ __device__ inline Smem smem_layout(char *base, int cache_rows, int sil, int spkcache_len) {
    Smem m;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char *p = base + off;
        off += (bytes + 15) & ~size_t(15);
        return p;
    };
    const size_t n = (size_t)(cache_rows + sil) * kSpeakers;
    m.scores = reinterpret_cast<float *>(take((size_t)cache_rows * kSpeakers * sizeof(float)));
    m.perm = reinterpret_cast<float *>(take(n * sizeof(float)));
    m.flag = reinterpret_cast<int *>(take(n * sizeof(int)));
    m.slot = reinterpret_cast<int *>(take((size_t)spkcache_len * sizeof(int)));
    m.scan = reinterpret_cast<int *>(take((kThreads + 1) * sizeof(int)));
    m.bytes = off;
    return m;
}

__device__ __forceinline__ int ring(int head, int j, int rows) {
    const int r = head + j;
    return r >= rows ? r - rows : r;
}

__device__ __forceinline__ void copy_row4(float *dst, const float *src) {   // 512 floats, 16-byte aligned, by the CTA
    for (int q = threadIdx.x; q < kDims / 4; q += kThreads)
        reinterpret_cast<float4 *>(dst)[q] = reinterpret_cast<const float4 *>(src)[q];
}

// Per-speaker top-k boost (boostTopKScores): every (frame, speaker) with a finite rank below k gains scale * ln2.
__device__ void boost_top_k(float *scores, int *flag, int L, int k, float scale) {
    if (k <= 0) return;
    for (int i = threadIdx.x; i < L * kSpeakers; i += kThreads) {
        const float v = scores[i];
        int kept = 0;
        if (v != -INFINITY) {
            const int spk = i & 3;
            kept = rank_until([&](int g) { return scores[g * kSpeakers + spk]; }, L, v, i >> 2, k, true) < k;
        }
        flag[i] = kept;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < L * kSpeakers; i += kThreads)
        if (flag[i]) scores[i] = boost(scores[i], scale);
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) sortformer_update_kernel(Config c, Arena a, const UpdateJob *__restrict__ jobs,
                                                                      const float *__restrict__ embs,
                                                                      const float *__restrict__ preds, float *state,
                                                                      long long *silence, float *confirmed,
                                                                      float *tentative) {
    extern __shared__ __align__(16) char smem_raw[];
    __shared__ int s_pos[kSpeakers];
    __shared__ long long s_silence;
    const UpdateJob J = jobs[blockIdx.x];
    const int tid = threadIdx.x;
    const int FR = c.fifo_rows();
    float *st = state + J.state;
    float *fifo = st + a.fifo, *fifo_p = st + a.fifo_preds, *mean = st + a.mean;
    float *cache = st + a.cache_at(J.parity), *cache_p = st + a.cache_preds_at(J.parity);
    const float *E = embs + J.emb, *P = preds + J.pred;

    // fifoPreds <- the fresh predictions of the FIFO rows (:47-55); append the core rows (:96-104); outputs (:73-94)
    const int chunk_start = J.spk_len + J.fifo_len + J.lc;
    for (int i = tid; i < J.fifo_len * kSpeakers; i += kThreads)
        fifo_p[ring(J.fifo_head, i >> 2, FR) * kSpeakers + (i & 3)] = P[(J.spk_len + (i >> 2)) * kSpeakers + (i & 3)];
    for (int j = 0; j < J.core; ++j) {
        float *dst = fifo + (size_t)ring(J.fifo_head, J.fifo_len + j, FR) * kDims;
        const float *src = E + (size_t)(J.lc + j) * kDims;
        for (int d = tid; d < kDims; d += kThreads) dst[d] = src[d];
    }
    for (int i = tid; i < J.core * kSpeakers; i += kThreads) {
        const float v = P[chunk_start * kSpeakers + i];
        fifo_p[ring(J.fifo_head, J.fifo_len + (i >> 2), FR) * kSpeakers + (i & 3)] = v;
        confirmed[J.confirmed + i] = v;
    }
    for (int i = tid; i < J.rc * kSpeakers; i += kThreads)
        tentative[J.tentative + i] = P[(chunk_start + J.core) * kSpeakers + i];
    if (J.pop == 0) return;
    // the count is read once, before the barrier, so that thread 0's write-back below can never be seen by a thread
    // that has not started its pass yet
    if (tid == 0) s_silence = silence[J.silence];
    __syncthreads();

    // updateSilenceProfile (:175-212): each thread owns dimensions, frames in order
    long long n = s_silence;
    for (int j = 0; j < J.pop; ++j) {
        const int r = ring(J.fifo_head, j, FR);
        if (prob_sum(fifo_p + r * kSpeakers) < c.silence_threshold) {
            const float nf = (float)n;
            for (int d = tid; d < kDims; d += kThreads) mean[d] = mean_step(mean[d], fifo[(size_t)r * kDims + d], nf);
            ++n;
        }
    }
    if (tid == 0) silence[J.silence] = n;
    // the popped rows join the speaker cache and its predictions (:135-147); the first compression takes the model's
    // predictions of the cache rows in front of them (:151-158)
    for (int j = 0; j < J.pop; ++j) copy_row4(cache + (size_t)(J.spk_len + j) * kDims, fifo + (size_t)ring(J.fifo_head, j, FR) * kDims);
    for (int i = tid; i < J.pop * kSpeakers; i += kThreads)
        cache_p[J.spk_len * kSpeakers + i] = fifo_p[ring(J.fifo_head, i >> 2, FR) * kSpeakers + (i & 3)];
    if (J.init_preds)
        for (int i = tid; i < J.spk_len * kSpeakers; i += kThreads) cache_p[i] = P[i];
    if (!J.compress) return;
    __syncthreads();

    // ---- compressSpkcache (:220-305)
    const int L = J.spk_len + J.pop, sil = c.sil_per_spk, F = L + sil, N = F * kSpeakers, K = c.spkcache_len;
    const Smem m = smem_layout(smem_raw, c.cache_rows(), sil, K);
    if (tid < kSpeakers) s_pos[tid] = 0;
    for (int f = tid; f < L; f += kThreads) frame_scores(cache_p + f * kSpeakers, c.pred_score_threshold, m.scores + f * kSpeakers);
    __syncthreads();
    {
        int cnt[kSpeakers] = {0, 0, 0, 0};
        for (int i = tid; i < L * kSpeakers; i += kThreads) cnt[i & 3] += positive_score(cache_p[i], m.scores[i]) ? 1 : 0;
        for (int k = 0; k < kSpeakers; ++k)
            if (cnt[k]) atomicAdd(&s_pos[k], cnt[k]);
    }
    __syncthreads();
    for (int i = tid; i < L * kSpeakers; i += kThreads)
        m.scores[i] = disable_and_boost(cache_p[i], m.scores[i], s_pos[i & 3], c.min_pos, (i >> 2) >= K, c.scores_boost_latest);
    __syncthreads();
    boost_top_k(m.scores, m.flag, L, c.strong_k, 2.0f);
    boost_top_k(m.scores, m.flag, L, c.weak_k, 1.0f);

    // getTopKIndices (:465-578) over permuted = spk * F + frame, placeholders +inf
    for (int p = tid; p < N; p += kThreads) {
        const int spk = p / F, f = p - spk * F;
        m.perm[p] = f < L ? m.scores[f * kSpeakers + spk] : INFINITY;
    }
    for (int r = tid; r < K; r += kThreads) m.slot[r] = -1;
    __syncthreads();
    for (int p = tid; p < N; p += kThreads) {
        const float v = m.perm[p];
        const float *perm = m.perm;
        m.flag[p] = rank_until([&](int q) { return perm[q]; }, N, v, p, K, false) < K && kept_index(v, p) != kMaxIndex;
    }
    __syncthreads();
    // ascending order of the kept real indices: an exclusive prefix sum over the flags, contiguous per thread
    const int per = (N + kThreads - 1) / kThreads, lo = min(N, tid * per), hi = min(N, lo + per);
    int own = 0;
    for (int p = lo; p < hi; ++p) own += m.flag[p];
    m.scan[tid + 1] = own;
    __syncthreads();
    if (tid == 0) {
        m.scan[0] = 0;
        for (int t = 1; t <= kThreads; ++t) m.scan[t] += m.scan[t - 1];
    }
    __syncthreads();
    for (int p = lo, pos = m.scan[tid]; p < hi; ++p) {
        if (!m.flag[p]) continue;
        const int f = p % F;
        if (pos < K) m.slot[pos] = f < L ? f : -1;   // frames >= F - sil are the placeholders: disabled
        ++pos;
    }
    __syncthreads();

    // gather into the other cache: a disabled slot takes the silence mean and zero predictions (:273-300)
    float *out = st + a.cache_at(J.parity ^ 1), *out_p = st + a.cache_preds_at(J.parity ^ 1);
    for (int r = 0; r < K; ++r) {
        const int f = m.slot[r];
        copy_row4(out + (size_t)r * kDims, f >= 0 ? cache + (size_t)f * kDims : mean);
    }
    for (int i = tid; i < K * kSpeakers; i += kThreads) {
        const int f = m.slot[i >> 2];
        out_p[i] = f >= 0 ? cache_p[f * kSpeakers + (i & 3)] : 0.0f;
    }
}

// rows [0, spkcache_len) of a session's spkcache tensor, then [0, fifo_len) of its fifo tensor, zero past the lengths.
// Sessions on grid x (up to 2^31 - 1 of them), rows on grid y, a CTA striding over rows when there are more than y.
__global__ void __launch_bounds__(128) sortformer_inputs_kernel(Config c, Arena a, const InputJob *__restrict__ jobs,
                                                                 const float *__restrict__ state, float *spkcache,
                                                                 float *fifo) {
    const InputJob J = jobs[blockIdx.x];
    const size_t session = blockIdx.x;
    const float *st = state + J.state;
    for (int r = blockIdx.y; r < c.spkcache_len + c.fifo_len; r += gridDim.y) {
        const float *src = nullptr;
        float *dst;
        if (r < c.spkcache_len) {
            dst = spkcache + (session * c.spkcache_len + r) * kDims;
            if (r < J.spk_len) src = st + a.cache_at(J.parity) + (size_t)r * kDims;
        } else {
            const int fr = r - c.spkcache_len;
            dst = fifo + (session * c.fifo_len + fr) * kDims;
            if (fr < J.fifo_len) src = st + a.fifo + (size_t)ring(J.fifo_head, fr, c.fifo_rows()) * kDims;
        }
        for (int d = threadIdx.x; d < kDims; d += 128) dst[d] = src ? src[d] : 0.0f;
    }
}

} // namespace

size_t update_smem_bytes(const Config &c) { return smem_layout(nullptr, c.cache_rows(), c.sil_per_spk, c.spkcache_len).bytes; }

int set_update_smem(const Config &c) {
    const size_t bytes = update_smem_bytes(c);
    if (bytes > kMaxDynamicSmem) {
        fa::set_error("sortformer: the compression needs %zu bytes of shared memory (limit %zu): lower max_core_frames, "
                      "fifoLen or spkcacheLen", bytes, kMaxDynamicSmem);
        return FA_INVALID_ARGUMENT;
    }
    // the attribute belongs to the kernel, not to the handle: every handle sets the same ceiling, so a handle created
    // later can never lower it below what an earlier one launches with
    FA_CUDA_TRY(cudaFuncSetAttribute(sortformer_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kMaxDynamicSmem));
    return FA_OK;
}

int launch_update(const Config &c, const Arena &a, const UpdateJob *d_jobs, int count, const float *embs, const float *preds,
                  float *state, long long *silence, float *confirmed, float *tentative, cudaStream_t s) {
    FA_CUDA_TRY(fa::launch(sortformer_update_kernel, count, kThreads, update_smem_bytes(c), s, c, a, d_jobs, embs, preds,
                           state, silence, confirmed, tentative));
    return FA_OK;
}

int launch_inputs(const Config &c, const Arena &a, const InputJob *d_jobs, int count, const float *state, float *spkcache,
                  float *fifo, cudaStream_t s) {
    const unsigned rows = (unsigned)std::min(c.spkcache_len + c.fifo_len, 65535);
    FA_CUDA_TRY(fa::launch(sortformer_inputs_kernel, dim3((unsigned)count, std::max(rows, 1u)), 128, 0, s, c, a, d_jobs,
                           state, spkcache, fifo));
    return FA_OK;
}

} // namespace sortformer
} // namespace fa
