// StyleTTS2 synthesis glue on the GPU (styletts2.h, styletts2_core.cuh).  Kernels (requests on blockIdx.x):
//   styletts2_sampler_kernel    bert's padded tokens and attention mask, and the fused sampler's 5 x 256 noise
//   styletts2_style_kernel      blendStyle
//   styletts2_durations_kernel  one CTA per request: roundDurations, one thread per token, and the prefix sum of the
//                               durations into the request's frame starts
//   styletts2_expand_kernel     the alignment matmul, the transpose and the HiFi-GAN shift of d and t_en in one pass:
//                               a CTA writes 64 frames x 32 channels of en or asr, coalesced along the frames.  d is
//                               token-major, so its rows for the tile's tokens go through a shared-memory tile; t_en is
//                               channel-major and is read along its rows directly.
#include "styletts2.h"

#include <algorithm>
#include <cstring>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace styletts2 {

namespace {

constexpr int kThreads = 256;
constexpr int kStarts = kMaxTokens + 1;   // a request's frame starts: starts[t] for t <= n, starts[n] = F
constexpr int kFrameTile = 64, kChannelTile = 32;

struct SamplerJob {
    long long src;   // the request's first id in the call's ids
    uint64_t s0;     // the noise state before the first draw
    int n, pad;
};

struct StyleJob {
    float alpha, beta;
};

struct AlignJob {
    long long logits, d, t;   // the request's offsets in logits, d and t_en
    int n, tok_at;            // its token count and its first duration in the packed durations
};

__global__ void __launch_bounds__(kThreads)
    styletts2_sampler_kernel(const SamplerJob *__restrict__ jobs, const int32_t *__restrict__ ids, int bucket,
                             int32_t *__restrict__ tokens, int32_t *__restrict__ mask, float *__restrict__ noise) {
    const int i = blockIdx.x;
    const SamplerJob J = jobs[i];
    const int k = blockIdx.y * kThreads + threadIdx.x;
    if (k < bucket) {
        const bool real = k < J.n;
        tokens[(size_t)i * bucket + k] = real ? ids[J.src + k] : 0;
        mask[(size_t)i * bucket + k] = real ? 1 : 0;
    }
    if (k < kNoiseFloats) noise[(size_t)i * kNoiseFloats + k] = luxtts::gaussian_at(J.s0, (uint64_t)k);
}

__global__ void __launch_bounds__(kRefSplit)
    styletts2_style_kernel(const StyleJob *__restrict__ jobs, const float *__restrict__ s_pred,
                           const float *__restrict__ ref_s, float *__restrict__ ref, float *__restrict__ s) {
    const int i = blockIdx.x, k = threadIdx.x;
    const StyleJob J = jobs[i];
    const float *P = s_pred + (size_t)i * kStyleDim, *R = ref_s + (size_t)i * kStyleDim;
    ref[(size_t)i * kRefSplit + k] = blend(J.alpha, P[k], R[k]);
    s[(size_t)i * kRefSplit + k] = blend(J.beta, P[kRefSplit + k], R[kRefSplit + k]);
}

__global__ void __launch_bounds__(kMaxTokens)
    styletts2_durations_kernel(const AlignJob *__restrict__ jobs, const float *__restrict__ logits,
                               long long logit_row, int channels, long long *__restrict__ starts,
                               long long *__restrict__ frames, int *__restrict__ flags, int *__restrict__ durations) {
    __shared__ long long scan[kMaxTokens];
    const int i = blockIdx.x, t = threadIdx.x;
    const AlignJob J = jobs[i];
    const int dur = t < J.n ? duration_of(logits + J.logits + t * logit_row, channels) : 0;
    const int nan = __syncthreads_or(dur < 0);
    scan[t] = dur < 0 ? 0 : dur;
    __syncthreads();
    for (int s = 1; s < kMaxTokens; s <<= 1) {   // inclusive prefix sum, Hillis-Steele
        const long long v = t >= s ? scan[t - s] : 0;
        __syncthreads();
        scan[t] += v;
        __syncthreads();
    }
    long long *S = starts + (size_t)i * kStarts;
    if (t < J.n) {
        S[t + 1] = scan[t];
        durations[J.tok_at + t] = dur;
    }
    if (t == 0) {
        S[0] = 0;
        frames[i] = scan[J.n - 1];
        flags[i] = nan;
    }
}

__global__ void __launch_bounds__(kThreads)
    styletts2_expand_kernel(const AlignJob *__restrict__ jobs, const long long *__restrict__ starts,
                            const float *__restrict__ d, long long d_row, int d_channels, const float *__restrict__ t_en,
                            long long t_row, int t_channels, long long frame_stride, int en_tiles,
                            float *__restrict__ en, float *__restrict__ asr) {
    __shared__ int tok[kFrameTile];                       // the token of each frame of the tile, -1 from F on
    __shared__ float tile[kFrameTile][kChannelTile + 1];  // d's rows for the tile's tokens
    const int i = blockIdx.x;
    const AlignJob J = jobs[i];
    const long long *S = starts + (size_t)i * kStarts;
    const long long F = S[J.n], f0 = (long long)blockIdx.y * kFrameTile;
    if (threadIdx.x < kFrameTile) {
        const long long f = f0 + threadIdx.x;
        tok[threadIdx.x] = f < F ? token_at(S, J.n, f > 0 ? f - 1 : 0) : -1;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int fl = (warp & 1) * 32 + lane;   // this thread's frame in the tile; warps 2k and 2k+1 share channels
    const long long f = f0 + fl;
    const int tk = tok[fl];
    if ((int)blockIdx.z < en_tiles) {
        const int c0 = blockIdx.z * kChannelTile, t0 = tok[0];
        if (t0 >= 0) {
            const int t1 = tok[F - f0 < kFrameTile ? (int)(F - f0) - 1 : kFrameTile - 1];
            for (int r = warp; r <= t1 - t0; r += kThreads / 32) {   // coalesced along d's channels
                const int c = c0 + lane;
                tile[r][lane] = c < d_channels ? d[J.d + (long long)(t0 + r) * d_row + c] : 0.0f;
            }
        }
        __syncthreads();
        if (f >= frame_stride) return;
        for (int k = warp >> 1; k < kChannelTile && c0 + k < d_channels; k += kThreads / 64)
            en[((size_t)i * d_channels + c0 + k) * frame_stride + f] = tk >= 0 ? expanded(tile[tk - t0][k]) : 0.0f;
    } else {
        const int c0 = (blockIdx.z - en_tiles) * kChannelTile;
        if (f >= frame_stride) return;
        for (int k = warp >> 1; k < kChannelTile && c0 + k < t_channels; k += kThreads / 64) {
            const int c = c0 + k;
            asr[((size_t)i * t_channels + c) * frame_stride + f] =
                tk >= 0 ? expanded(t_en[J.t + (long long)c * t_row + tk]) : 0.0f;
        }
    }
}

unsigned tiles(long long n, long long per) { return (unsigned)std::max(1LL, (n + per - 1) / per); }

template <typename Job> int upload_jobs(CallContext &C, const std::vector<Job> &jobs) {
    const size_t bytes = jobs.size() * sizeof(Job);
    int st = C.stage.reserve(bytes);
    if (st != FA_OK) return st;
    std::memcpy(C.stage.host.data(), jobs.data(), bytes);
    return C.stage.upload(bytes, C.stream);
}

} // namespace

int sampler_inputs(CallContext &C, int count, const int32_t *token_ids, const int64_t *offsets, const uint64_t *seeds,
                   int bucket, bool device, int32_t *tokens, int32_t *mask, float *noise) {
    std::vector<SamplerJob> jobs((size_t)count);
    for (int i = 0; i < count; ++i)
        jobs[i] = SamplerJob{offsets[i] - offsets[0], luxtts::seed_state(seeds[i]), (int)(offsets[i + 1] - offsets[i]), 0};
    int st = upload_jobs(C, jobs);
    if (st != FA_OK) return st;
    HostStaging H(!device, C.stream);
    const int32_t *k_ids;
    int32_t *k_tokens, *k_mask;
    float *k_noise;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_ids = l.in(token_ids + offsets[0], (size_t)(offsets[count] - offsets[0]));
        k_tokens = l.out(tokens, (size_t)count * bucket);
        k_mask = l.out(mask, (size_t)count * bucket);
        k_noise = l.out(noise, (size_t)count * kNoiseFloats);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(styletts2_sampler_kernel, dim3((unsigned)count, tiles(kNoiseFloats, kThreads)), kThreads, 0,
                       C.stream, static_cast<const SamplerJob *>(C.stage.device.data()), k_ids, bucket, k_tokens,
                       k_mask, k_noise));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int style(CallContext &C, int count, const float *s_pred, const float *ref_s, const float *alphas, const float *betas,
          bool device, float *ref, float *s) {
    std::vector<StyleJob> jobs((size_t)count);
    for (int i = 0; i < count; ++i) jobs[i] = StyleJob{alphas[i], betas[i]};
    int st = upload_jobs(C, jobs);
    if (st != FA_OK) return st;
    HostStaging H(!device, C.stream);
    const float *k_p, *k_r;
    float *k_ref, *k_s;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_p = l.in(s_pred, (size_t)count * kStyleDim);
        k_r = l.in(ref_s, (size_t)count * kStyleDim);
        k_ref = l.out(ref, (size_t)count * kRefSplit);
        k_s = l.out(s, (size_t)count * kRefSplit);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(styletts2_style_kernel, dim3((unsigned)count), kRefSplit, 0, C.stream,
                       static_cast<const StyleJob *>(C.stage.device.data()), k_p, k_r, k_ref, k_s));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int align(CallContext &C, const AlignArgs &a, bool device, const char *where) {
    const int count = a.count;
    std::vector<AlignJob> jobs((size_t)count);
    int total = 0;
    for (int i = 0; i < count; ++i) {
        jobs[i] = AlignJob{i * a.logit_request, i * a.d_request, i * a.t_request, a.token_counts[i], total};
        total += a.token_counts[i];
    }
    const int n_last = a.token_counts[count - 1];
    int st = upload_jobs(C, jobs);
    if (st != FA_OK) return st;
    long long *d_starts, *d_frames;
    int *d_flags, *d_durs;
    st = carve_arena(C.scratch, [&](Carver &c) {
        d_starts = c.take<long long>((size_t)count * kStarts);
        d_frames = c.take<long long>((size_t)count);   // frames, flags and durations come back in one copy
        d_flags = c.take<int>((size_t)count);
        d_durs = c.take<int>((size_t)total);
    });
    if (st != FA_OK) return st;
    const size_t back = (size_t)(reinterpret_cast<char *>(d_durs + total) - reinterpret_cast<char *>(d_frames));
    st = C.h_buf.grow(back);
    if (st != FA_OK) return st;
    HostStaging H(!device, C.stream);
    const float *k_logits, *k_d, *k_t;
    float *k_en, *k_asr;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_logits = l.in(a.logits, (size_t)((count - 1) * a.logit_request + (n_last - 1) * a.logit_row + a.channels));
        k_d = l.in(a.d, (size_t)((count - 1) * a.d_request + (n_last - 1) * a.d_row + a.d_channels));
        k_t = l.in(a.t_en, (size_t)((count - 1) * a.t_request + (a.t_channels - 1) * a.t_row + n_last));
        k_en = l.out(a.en, (size_t)count * a.d_channels * a.frame_stride);
        k_asr = l.out(a.asr, (size_t)count * a.t_channels * a.frame_stride);
    });
    if (st != FA_OK) return st;
    const auto *d_jobs = static_cast<const AlignJob *>(C.stage.device.data());
    FA_CUDA_TRY(launch(styletts2_durations_kernel, dim3((unsigned)count), kMaxTokens, 0, C.stream, d_jobs, k_logits,
                       a.logit_row, a.channels, d_starts, d_frames, d_flags, d_durs));
    char *h = static_cast<char *>(C.h_buf.data());
    FA_CUDA_TRY(cudaMemcpyAsync(h, d_frames, back, cudaMemcpyDeviceToHost, C.stream));
    FA_CUDA_TRY(cudaStreamSynchronize(C.stream));
    const auto *h_frames = reinterpret_cast<const long long *>(h);
    const auto *h_flags = reinterpret_cast<const int *>(h + (reinterpret_cast<char *>(d_flags) - reinterpret_cast<char *>(d_frames)));
    const auto *h_durs = reinterpret_cast<const int *>(h + (reinterpret_cast<char *>(d_durs) - reinterpret_cast<char *>(d_frames)));

    int nan = -1, over = -1;
    for (int i = 0; i < count; ++i) {
        if (h_flags[i] && nan < 0) nan = i;
        if (h_frames[i] > a.frame_stride && over < 0) over = i;
    }
    if (nan >= 0) {
        for (int i = 0; i < count; ++i) a.reasons[i] = h_flags[i] ? kNonfiniteDuration : kOk;
        set_error("%s: request %d has a NaN duration logit (see reasons)", where, nan);
        return FA_INVALID_ARGUMENT;
    }
    for (int i = 0; i < count; ++i) a.reasons[i] = kOk;
    if (over >= 0) {
        for (int i = 0; i < count; ++i) a.frames[i] = h_frames[i];
        set_error("%s: request %d has %lld frames, frame_stride is %lld", where, over, h_frames[over], a.frame_stride);
        return FA_OUTPUT_TOO_SMALL;
    }
    const int en_tiles = (int)tiles(a.d_channels, kChannelTile);
    FA_CUDA_TRY(launch(styletts2_expand_kernel,
                       dim3((unsigned)count, tiles(a.frame_stride, kFrameTile),
                            en_tiles + tiles(a.t_channels, kChannelTile)),
                       kThreads, 0, C.stream, d_jobs, d_starts, k_d, a.d_row, a.d_channels, k_t, a.t_row, a.t_channels,
                       a.frame_stride, en_tiles, k_en, k_asr));
    FA_CUDA_TRY(H.finish());
    for (int i = 0; i < count; ++i) a.frames[i] = h_frames[i];
    if (a.durations) std::memcpy(a.durations, h_durs, (size_t)total * sizeof(int32_t));
    return FA_OK;
}

} // namespace styletts2
} // namespace fa
