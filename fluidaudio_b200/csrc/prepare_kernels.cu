// The offline diarizer's prepare stage on the GPU (interface and reference lines: prepare_plan.h; arithmetic:
// prepare_core.cuh).
//
//   seg_windows_kernel      gathers analysis windows (and the extractor's fbank windows) from the audio, zero tail
//   seg_decode_kernel       one thread per frame: log-probabilities, binary speaker weights, class histogram, speech frames
//   embedding_mask_kernel   one CTA per chunk: overlap frames, per local speaker the base / clean sums, the skip and
//                           fallback decisions, first / last active frame and the resampled mask's energy
//   embedding_pack_kernel   one CTA per chunk: its first slot from the per-chunk counts (a prefix sum, so entries are
//                           packed chunk-major, speaker-minor as the reference emits them), then the rows of its entries
//   mask_reuse_kernel       one warp per (FBANK batch, local speaker): the mask-similarity skip strategy
//   weight_resample_kernel  WeightInterpolation.resample2D on packed rows
//
// fa_seg_decode is one launch; fa_embedding_plan is two, three with the skip strategy, whatever the chunk count.
#include "prepare_plan.h"

#include "call_context.h"
#include "prepare_core.cuh"

#include <algorithm>
#include <climits>
#include <cmath>

namespace fa {
namespace prepare {

namespace {

constexpr int kThreads = kSumLanes;
constexpr size_t kMaxDynamicSmem = 200 * 1024;

struct ChunkDesc {
    double offset;   // resolved chunkOffsetSeconds
    int active;      // the chunk reaches the embedding stage (it has audio)
    int pad;
};

struct EntryMeta {
    int flags;       // bit 0 emitted, bit 1 clean mask, bit 2 fallback
    int first, last;
    float mask_sum;
};
enum : int { kEmit = 1, kClean = 2, kFallback = 4 };

// ---------------------------------------------------------------------------------------------- windows
__global__ void __launch_bounds__(kThreads) seg_windows_kernel(const float *__restrict__ audio,
                                                                const WindowDesc *__restrict__ desc, long long row_len,
                                                                float *__restrict__ out) {
    const WindowDesc d = desc[blockIdx.x];
    const float *src = audio + d.start;
    float *dst = out + (size_t)blockIdx.x * (size_t)row_len;
    const long long stride = (long long)gridDim.y * kThreads;
    const long long t = (long long)blockIdx.y * kThreads + threadIdx.x;
    long long scalar_from = 0;
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
        const long long quads = row_len / 4, full = d.copy / 4;   // quads below `full` lie wholly inside the audio
        for (long long q = t; q < quads; q += stride) {
            float4 v;
            if (q < full) {
                v = reinterpret_cast<const float4 *>(src)[q];
            } else {
                const long long i = q * 4;
                v.x = i < d.copy ? src[i] : 0.0f;
                v.y = i + 1 < d.copy ? src[i + 1] : 0.0f;
                v.z = i + 2 < d.copy ? src[i + 2] : 0.0f;
                v.w = 0.0f;
            }
            reinterpret_cast<float4 *>(dst)[q] = v;
        }
        scalar_from = quads * 4;
    }
    for (long long i = scalar_from + t; i < row_len; i += stride) dst[i] = i < d.copy ? src[i] : 0.0f;
}

// ---------------------------------------------------------------------------------------------- decode
// Shared memory: kThreads rows of logits with an odd stride (so that the per-thread rows fall in distinct banks), then
// kThreads x 3 weights; both are filled and drained with consecutive threads on consecutive addresses.
__global__ void __launch_bounds__(kThreads) seg_decode_kernel(const float *__restrict__ logits, long long total_frames,
                                                               int classes, float onset, float *__restrict__ log_probs,
                                                               float *__restrict__ weights,
                                                               unsigned long long *__restrict__ tallies) {
    extern __shared__ float sm[];
    __shared__ unsigned s_tally[kPowersetClasses + 1];
    const int stride = classes | 1;
    float *rows = sm, *w = sm + kThreads * stride;
    const long long f0 = (long long)blockIdx.x * kThreads;
    const int nf = (int)min((long long)kThreads, total_frames - f0);
    const int tid = threadIdx.x;
    if (tid <= kPowersetClasses) s_tally[tid] = 0;
    const float *src = logits + f0 * classes;
    for (int i = tid; i < nf * classes; i += kThreads) rows[(i / classes) * stride + i % classes] = src[i];
    __syncthreads();
    if (tid < nf) {
        float *row = rows + tid * stride;
        const FrameDecision d = decode_frame(row, classes, onset, row);
        if (d.best < kPowersetClasses) atomicAdd(&s_tally[d.best], 1u);
        if (d.speech) atomicAdd(&s_tally[kPowersetClasses], 1u);
        const unsigned who = powerset_speakers(min(d.best, kPowersetClasses - 1));
        for (int s = 0; s < kDecodeSpeakers; ++s) w[tid * kDecodeSpeakers + s] = (who >> s) & 1u ? 1.0f : 0.0f;
    }
    __syncthreads();
    if (log_probs) {
        float *dst = log_probs + f0 * classes;
        for (int i = tid; i < nf * classes; i += kThreads) dst[i] = rows[(i / classes) * stride + i % classes];
    }
    float *wdst = weights + f0 * kDecodeSpeakers;
    for (int i = tid; i < nf * kDecodeSpeakers; i += kThreads) wdst[i] = w[i];
    if (tid <= kPowersetClasses && s_tally[tid]) atomicAdd(&tallies[tid], (unsigned long long)s_tally[tid]);
}

// ---------------------------------------------------------------------------------------------- masks
// A chunk's [frames x speakers] weights and its overlap frames (:432-447) in shared memory.
__device__ void load_chunk(const float *__restrict__ w, int frames, int speakers, bool exclude, float *sw,
                           unsigned char *overlap) {
    for (int i = threadIdx.x; i < frames * speakers; i += kThreads) sw[i] = w[i];
    __syncthreads();
    for (int f = threadIdx.x; f < frames; f += kThreads) {
        int active = 0;
        for (int s = 0; s < speakers; ++s) active += sw[f * speakers + s] > kActiveThreshold ? 1 : 0;
        overlap[f] = exclude && active > 1;
    }
    __syncthreads();
}

struct ChunkSmem {
    float *w, *mask;
    unsigned char *overlap;
};
__device__ ChunkSmem chunk_smem(float *sm, int frames, int speakers) {
    ChunkSmem c;
    c.w = sm;
    c.mask = sm + frames * speakers;
    c.overlap = reinterpret_cast<unsigned char *>(c.mask + frames);
    return c;
}
size_t chunk_smem_bytes(int frames, int speakers) {
    return sizeof(float) * ((size_t)frames * speakers + frames) + frames;
}

struct MaskSums {
    float base, clean;
    int first_base, last_base, first_clean, last_clean;
};

// ordered_sum's order (prepare_core.cuh): each thread holds its lane's partial on entry, red[0] the total on return.
__device__ void fold_lanes(MaskSums *red) {
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        __syncthreads();
        if (threadIdx.x < h) {
            MaskSums a = red[threadIdx.x];
            const MaskSums b = red[threadIdx.x + h];
            a.base = f_add(a.base, b.base);
            a.clean = f_add(a.clean, b.clean);
            a.first_base = min(a.first_base, b.first_base);
            a.last_base = max(a.last_base, b.last_base);
            a.first_clean = min(a.first_clean, b.first_clean);
            a.last_clean = max(a.last_clean, b.last_clean);
            red[threadIdx.x] = a;
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) embedding_mask_kernel(const float *__restrict__ weights, int frames,
                                                                   int speakers, int exclude, int min_frames,
                                                                   int weight_frames, const ChunkDesc *__restrict__ desc,
                                                                   EntryMeta *__restrict__ meta,
                                                                   int *__restrict__ chunk_count, int *__restrict__ counters) {
    extern __shared__ float sm[];
    __shared__ MaskSums red[kThreads];
    const int c = blockIdx.x, tid = threadIdx.x;
    if (!desc[c].active) {   // the reference never evaluates a chunk without audio (:666-668)
        if (tid == 0) chunk_count[c] = 0;
        for (int s = tid; s < speakers; s += kThreads) meta[(size_t)c * speakers + s] = EntryMeta{0, 0, 0, 0.0f};
        return;
    }
    const ChunkSmem k = chunk_smem(sm, frames, speakers);
    load_chunk(weights + (size_t)c * frames * speakers, frames, speakers, exclude != 0, k.w, k.overlap);
    int emitted = 0, empty = 0, fallback = 0;
    for (int s = 0; s < speakers; ++s) {
        MaskSums a = {0.0f, 0.0f, INT_MAX, -1, INT_MAX, -1};
        for (int f = tid; f < frames; f += kThreads) {
            const float v = k.w[f * speakers + s], cv = k.overlap[f] ? 0.0f : v;
            a.base = f_add(a.base, v);
            a.clean = f_add(a.clean, cv);
            if (v > kActiveThreshold) {
                a.first_base = min(a.first_base, f);
                a.last_base = f;
            }
            if (cv > kActiveThreshold) {
                a.first_clean = min(a.first_clean, f);
                a.last_clean = f;
            }
        }
        red[tid] = a;
        fold_lanes(red);
        const MaskSums total = red[0];
        const MaskDecision d = mask_decide(total.base, total.clean, frames, min_frames);
        fallback += d.fallback;
        int emit = 0;
        if (d.candidate) {   // uniform over the CTA
            for (int f = tid; f < frames; f += kThreads)
                k.mask[f] = d.use_clean && k.overlap[f] ? 0.0f : k.w[f * speakers + s];
            __syncthreads();
            float e = 0.0f;
            for (int j = tid; j < weight_frames; j += kThreads) e = f_add(e, resample_at(k.mask, frames, weight_frames, j));
            red[tid].base = e;
            red[tid].clean = 0.0f;
            fold_lanes(red);
            emit = red[0].base <= 0.0f ? 0 : 1;   // maskEnergy <= 0 (:549)
        }
        empty += 1 - emit;
        emitted += emit;
        if (tid == 0) {
            const int first = d.use_clean ? total.first_clean : total.first_base;
            const int last = d.use_clean ? total.last_clean : total.last_base;
            EntryMeta m;
            m.flags = (emit ? kEmit : 0) | (d.use_clean ? kClean : 0) | (d.fallback ? kFallback : 0);
            m.first = first == INT_MAX ? 0 : first;   // firstIndex(where:) ?? 0, lastIndex(where:) ?? firstActive
            m.last = last < 0 ? m.first : last;
            m.mask_sum = d.mask_sum;
            meta[(size_t)c * speakers + s] = m;
        }
        __syncthreads();   // red and mask are rewritten for the next speaker
    }
    if (tid == 0) {
        chunk_count[c] = emitted;
        atomicAdd(&counters[0], speakers);
        if (empty) atomicAdd(&counters[1], empty);
        if (fallback) atomicAdd(&counters[2], fallback);
    }
}

struct PackTargets {
    PlanOutputs out;
    int *slot_of;       // [chunks x speakers] entry index, -1 when the pair is skipped
    int *entry_count;
};

__global__ void __launch_bounds__(kThreads) embedding_pack_kernel(const float *__restrict__ weights, int chunks, int frames,
                                                                   int speakers, int exclude, int weight_frames,
                                                                   double frame_duration,
                                                                   const ChunkDesc *__restrict__ desc,
                                                                   const EntryMeta *__restrict__ meta,
                                                                   const int *__restrict__ chunk_count, PackTargets t) {
    extern __shared__ float sm[];
    __shared__ int part[kThreads];
    const int c = blockIdx.x, tid = threadIdx.x;
    int before = 0;
    for (int i = tid; i < c; i += kThreads) before += chunk_count[i];
    part[tid] = before;
    for (int h = kThreads / 2; h > 0; h >>= 1) {
        __syncthreads();
        if (tid < h) part[tid] += part[tid + h];
    }
    __syncthreads();
    int slot = part[0];
    const int mine = chunk_count[c];
    if (c == chunks - 1 && tid == 0) *t.entry_count = slot + mine;
    if (mine == 0) {
        for (int s = tid; s < speakers; s += kThreads) t.slot_of[(size_t)c * speakers + s] = -1;
        return;
    }
    const ChunkSmem k = chunk_smem(sm, frames, speakers);
    load_chunk(weights + (size_t)c * frames * speakers, frames, speakers, exclude != 0, k.w, k.overlap);
    const double offset = desc[c].offset;
    for (int s = 0; s < speakers; ++s) {
        const EntryMeta m = meta[(size_t)c * speakers + s];
        if (!(m.flags & kEmit)) {
            if (tid == 0) t.slot_of[(size_t)c * speakers + s] = -1;
            continue;
        }
        if (tid == 0) {
            const PlanOutputs &o = t.out;
            t.slot_of[(size_t)c * speakers + s] = slot;
            if (o.chunk_index) o.chunk_index[slot] = c;
            if (o.speaker_index) o.speaker_index[slot] = s;
            if (o.start_frame) o.start_frame[slot] = m.first;
            if (o.end_frame) o.end_frame[slot] = m.last;
            if (o.start_time) o.start_time[slot] = frame_time(offset, m.first, frame_duration);
            if (o.end_time) o.end_time[slot] = frame_time(offset, m.last + 1, frame_duration);
            if (o.mask_sum) o.mask_sum[slot] = m.mask_sum;
            if (o.used_fallback) o.used_fallback[slot] = m.flags & kFallback ? 1 : 0;
            if (o.reuse_of) o.reuse_of[slot] = -1;
        }
        const bool clean = (m.flags & kClean) != 0;
        for (int f = tid; f < frames; f += kThreads) {
            const float v = clean && k.overlap[f] ? 0.0f : k.w[f * speakers + s];
            k.mask[f] = v;
            if (t.out.frame_weights) t.out.frame_weights[(size_t)slot * frames + f] = v;
        }
        __syncthreads();
        if (t.out.model_weights)
            for (int j = tid; j < weight_frames; j += kThreads)
                t.out.model_weights[(size_t)slot * weight_frames + j] = resample_at(k.mask, frames, weight_frames, j);
        __syncthreads();
        ++slot;
    }
}

// The skip strategy (:554-585, 632-639).  A warp owns local speaker s of one FBANK batch and walks the batch's chunks in
// order: an entry whose mask has cosine >= threshold with the mask that produced the cached embedding reuses that
// entry, any other entry becomes the cache.  The three dot products run lane-strided from 0 over the 32 lanes, which
// are then folded by a xor butterfly (vDSP_dotpr's order is closed; binary masks give exact integers in any order).
__global__ void __launch_bounds__(kThreads) mask_reuse_kernel(const int *__restrict__ active, int active_count, int batch,
                                                               int speakers, int frames, const int *__restrict__ slot_of,
                                                               const float *__restrict__ masks, float threshold,
                                                               int *__restrict__ reuse_of, int *__restrict__ counters) {
    const int warp = (int)((blockIdx.x * (unsigned)kThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    const int batches = (active_count + batch - 1) / batch;
    if (warp >= batches * speakers) return;
    const int b = warp / speakers, s = warp % speakers;
    int cached = -1, skipped = 0;
    const int end = min(active_count, (b + 1) * batch);
    for (int i = b * batch; i < end; ++i) {
        const int slot = slot_of[(size_t)active[i] * speakers + s];
        if (slot < 0) continue;
        if (cached >= 0) {
            const float *x = masks + (size_t)slot * frames, *y = masks + (size_t)cached * frames;
            float dot = 0.0f, nx = 0.0f, ny = 0.0f;
            for (int f = lane; f < frames; f += 32) {
                dot = f_add(dot, f_mul(x[f], y[f]));
                nx = f_add(nx, f_mul(x[f], x[f]));
                ny = f_add(ny, f_mul(y[f], y[f]));
            }
            for (int m = 16; m > 0; m >>= 1) {
                dot = f_add(dot, __shfl_xor_sync(0xffffffffu, dot, m));
                nx = f_add(nx, __shfl_xor_sync(0xffffffffu, nx, m));
                ny = f_add(ny, __shfl_xor_sync(0xffffffffu, ny, m));
            }
            if (mask_cosine(dot, nx, ny) >= threshold) {
                if (lane == 0 && reuse_of) reuse_of[slot] = cached;
                ++skipped;
                continue;
            }
        }
        cached = slot;
    }
    if (lane == 0 && skipped) atomicAdd(&counters[3], skipped);
}

__global__ void __launch_bounds__(kThreads) weight_resample_kernel(const float *__restrict__ rows, long long total,
                                                                    int in_len, int out_len, float *__restrict__ out) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
        const long long r = i / out_len;
        out[i] = resample_at(rows + r * in_len, in_len, out_len, (int)(i - r * out_len));
    }
}

// ---------------------------------------------------------------------------------------------- host side
template <typename Kernel> int allow_smem(Kernel kernel, size_t bytes, const char *what) {
    if (bytes > kMaxDynamicSmem) {
        set_error("%s: %zu bytes of shared memory per chunk exceed %zu", what, bytes, kMaxDynamicSmem);
        return FA_UNSUPPORTED;
    }
    if (bytes > 48 * 1024)
        FA_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return FA_OK;
}

} // namespace

bool seg_config_ok(const SegConfig &c) {
    return c.sample_rate > 0 && c.window_duration > 0.0 && c.step_ratio > 0.0 && c.step_ratio <= 1.0 &&
           (double)c.sample_rate * c.window_duration < 2147483648.0 && samples_per_window(c) >= 1;
}
long long samples_per_window(const SegConfig &c) { return (long long)((double)c.sample_rate * c.window_duration); }
long long samples_per_step(const SegConfig &c) {
    return std::max(1LL, (long long)((double)samples_per_window(c) * c.step_ratio));
}
long long window_count(long long total_samples, const SegConfig &c) {   // stride(from: 0, to: totalSamples, by: step)
    const long long step = samples_per_step(c);
    return total_samples <= 0 ? 0 : (total_samples + step - 1) / step;
}

double resolve_chunk_offset(const double *offsets, int offsets_count, int c, const SegConfig &cfg) {
    const double fallback = (double)c * cfg.window_duration;
    if (c >= offsets_count) return fallback;
    return std::isfinite(offsets[c]) ? offsets[c] : fallback;
}

WindowDesc embed_window(double chunk_offset, long long total_samples, const SegConfig &cfg, int audio_sample_count) {
    const double estimated = std::round(chunk_offset * (double)cfg.sample_rate);   // .rounded(): ties away from zero
    const long long start = estimated <= 0.0 ? 0 : (estimated >= (double)total_samples ? total_samples : (long long)estimated);
    const long long end = std::min(start + samples_per_window(cfg), total_samples);
    return WindowDesc{start, start < end ? std::min<long long>(end - start, audio_sample_count) : 0};
}

int gather_windows(CallContext &C, bool on_device, const float *audio, long long total_samples, const WindowDesc *desc,
                   int count, long long row_len, float *out) {
    const cudaStream_t s = C.stream;
    const size_t desc_bytes = (size_t)count * sizeof(WindowDesc);
    int st = C.stage.reserve(desc_bytes);
    if (st != FA_OK) return st;
    std::copy(desc, desc + count, static_cast<WindowDesc *>(C.stage.host.data()));
    if ((st = C.stage.upload(desc_bytes, s)) != FA_OK) return st;
    HostStaging H(!on_device, s);
    const float *d_audio;
    float *d_out;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_audio = l.in(audio, (size_t)total_samples);
        d_out = l.out(out, (size_t)count * (size_t)row_len);
    });
    if (st != FA_OK) return st;
    const unsigned tiles = (unsigned)std::min<long long>(16, (row_len + 4 * kThreads - 1) / (4 * kThreads));
    FA_CUDA_TRY(launch(seg_windows_kernel, dim3((unsigned)count, std::max(1u, tiles)), dim3(kThreads), 0, s, d_audio,
                       static_cast<const WindowDesc *>(C.stage.device.data()), row_len, d_out));
    FA_CUDA_TRY(H.back());
    FA_CUDA_TRY(cudaStreamSynchronize(s));
    return FA_OK;
}

int seg_decode(CallContext &C, bool on_device, const float *logits, int chunks, int frames, int classes, float onset,
               float *log_probs, float *speaker_weights, int64_t histogram[8], int64_t *speech_frames) {
    const cudaStream_t s = C.stream;
    const long long total = (long long)chunks * frames;
    const size_t in_floats = (size_t)total * classes;
    constexpr size_t kTallyBytes = (kPowersetClasses + 1) * sizeof(unsigned long long);
    int st = C.scratch.grow(kTallyBytes);
    if (st != FA_OK) return st;
    auto *tallies = static_cast<unsigned long long *>(C.scratch.data());
    FA_CUDA_TRY(cudaMemsetAsync(tallies, 0, kTallyBytes, s));
    HostStaging H(!on_device, s);
    const float *d_logits;
    float *d_lp, *d_w;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_logits = l.in(logits, in_floats);
        d_lp = l.out(log_probs, in_floats);
        d_w = l.out(speaker_weights, (size_t)total * kDecodeSpeakers);
    });
    if (st != FA_OK) return st;
    const size_t smem = sizeof(float) * kThreads * ((size_t)(classes | 1) + kDecodeSpeakers);
    FA_CUDA_TRY(launch(seg_decode_kernel, dim3((unsigned)((total + kThreads - 1) / kThreads)), dim3(kThreads), smem, s,
                       d_logits, total, classes, onset, d_lp, d_w, tallies));
    FA_CUDA_TRY(H.back());
    unsigned long long host_tallies[kPowersetClasses + 1];
    FA_CUDA_TRY(cudaMemcpyAsync(host_tallies, tallies, kTallyBytes, cudaMemcpyDeviceToHost, s));
    FA_CUDA_TRY(cudaStreamSynchronize(s));
    for (int k = 0; histogram && k < kPowersetClasses; ++k) histogram[k] = (int64_t)host_tallies[k];
    if (speech_frames) *speech_frames = (int64_t)host_tallies[kPowersetClasses];
    return FA_OK;
}

int embedding_plan(CallContext &C, bool on_device, const float *speaker_weights, int chunks, int frames, int speakers,
                   const double *chunk_offsets, int offsets_count, double frame_duration, long long total_samples,
                   const SegConfig &seg, const PlanConfig &plan, const PlanOutputs &out, int32_t *entry_count,
                   int64_t counters[4]) {
    const cudaStream_t s = C.stream;
    const size_t pairs = (size_t)chunks * speakers, w_floats = pairs * frames;
    const bool reuse = plan.skip_threshold >= 0.0f;

    // resolveFrameDuration (:370-379), requiredMinFrames (:381-387)
    if (!(frame_duration > 0.0)) frame_duration = seg.window_duration / (double)std::max(1, frames);
    int min_frames = 1;
    if (frame_duration > 0.0) {
        const double need = std::ceil(plan.min_segment_duration / frame_duration);
        min_frames = need >= (double)INT_MAX ? INT_MAX : std::max(1, (int)need);
    }

    // per chunk: its offset and whether it reaches the embedding stage; then the reaching chunks in order (FBANK batches
    // are counted over those)
    const size_t desc_bytes = ((size_t)chunks * sizeof(ChunkDesc) + 255) & ~size_t(255);
    int st = C.stage.reserve(desc_bytes + (size_t)chunks * sizeof(int));
    if (st != FA_OK) return st;
    auto *desc = static_cast<ChunkDesc *>(C.stage.host.data());
    int *active = reinterpret_cast<int *>(static_cast<char *>(C.stage.host.data()) + desc_bytes);
    int active_count = 0;
    for (int c = 0; c < chunks; ++c) {
        desc[c].offset = resolve_chunk_offset(chunk_offsets, offsets_count, c, seg);
        desc[c].active = embed_window(desc[c].offset, total_samples, seg, plan.audio_sample_count).copy > 0 ? 1 : 0;
        desc[c].pad = 0;
        if (desc[c].active) active[active_count++] = c;
    }
    if ((st = C.stage.upload(desc_bytes + (size_t)chunks * sizeof(int), s)) != FA_OK) return st;
    const auto *d_desc = static_cast<const ChunkDesc *>(C.stage.device.data());
    const int *d_active = reinterpret_cast<const int *>(static_cast<const char *>(C.stage.device.data()) + desc_bytes);

    // the host-buffer call stages the weights and packs into device arrays of full capacity, then copies the emitted
    // entries back
    HostStaging H(!on_device, s);
    PlanOutputs d;
    const float *d_weights;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_weights = l.in(speaker_weights, w_floats);
        d.chunk_index = l.out(out.chunk_index, pairs);
        d.speaker_index = l.out(out.speaker_index, pairs);
        d.start_frame = l.out(out.start_frame, pairs);
        d.end_frame = l.out(out.end_frame, pairs);
        d.start_time = l.out(out.start_time, pairs);
        d.end_time = l.out(out.end_time, pairs);
        d.mask_sum = l.out(out.mask_sum, pairs);
        d.used_fallback = l.out(out.used_fallback, pairs);
        d.reuse_of = l.out(out.reuse_of, pairs);
        d.frame_weights = l.out(out.frame_weights, pairs * frames);
        d.model_weights = l.out(out.model_weights, pairs * plan.weight_frames);
    });
    if (st != FA_OK) return st;

    EntryMeta *meta = nullptr;
    int *chunk_count = nullptr, *slot_of = nullptr, *tallies = nullptr;   // tallies: 4 counters, then the entry count
    float *own_masks = nullptr;
    st = carve_arena(C.scratch, [&](Carver &c) {
        meta = c.take<EntryMeta>(pairs);
        chunk_count = c.take<int>(chunks);
        slot_of = c.take<int>(pairs);
        tallies = c.take<int>(5);
        if (reuse && !d.frame_weights) own_masks = c.take<float>(pairs * frames);   // the skip strategy compares masks
    });
    if (st != FA_OK) return st;
    if (own_masks) d.frame_weights = own_masks;
    FA_CUDA_TRY(cudaMemsetAsync(tallies, 0, 5 * sizeof(int), s));

    const size_t smem = chunk_smem_bytes(frames, speakers);
    if ((st = allow_smem(embedding_mask_kernel, smem, "fa_embedding_plan")) != FA_OK) return st;
    if ((st = allow_smem(embedding_pack_kernel, smem, "fa_embedding_plan")) != FA_OK) return st;
    FA_CUDA_TRY(launch(embedding_mask_kernel, dim3((unsigned)chunks), dim3(kThreads), smem, s, d_weights, frames, speakers,
                       plan.exclude_overlap ? 1 : 0, min_frames, plan.weight_frames, d_desc, meta, chunk_count, tallies));
    FA_CUDA_TRY(launch(embedding_pack_kernel, dim3((unsigned)chunks), dim3(kThreads), smem, s, d_weights, chunks, frames,
                       speakers, plan.exclude_overlap ? 1 : 0, plan.weight_frames, frame_duration, d_desc,
                       static_cast<const EntryMeta *>(meta), static_cast<const int *>(chunk_count),
                       PackTargets{d, slot_of, tallies + 4}));
    if (reuse && active_count > 0) {
        const int batch = std::max(1, plan.fbank_batch);
        const long long warps = (long long)((active_count + batch - 1) / batch) * speakers;
        FA_CUDA_TRY(launch(mask_reuse_kernel, dim3((unsigned)((warps * 32 + kThreads - 1) / kThreads)), dim3(kThreads), 0, s,
                           d_active, active_count, batch, speakers, frames, static_cast<const int *>(slot_of),
                           static_cast<const float *>(d.frame_weights), plan.skip_threshold, d.reuse_of, tallies));
    }
    int host_tallies[5];
    FA_CUDA_TRY(cudaMemcpyAsync(host_tallies, tallies, sizeof(host_tallies), cudaMemcpyDeviceToHost, s));
    FA_CUDA_TRY(cudaStreamSynchronize(s));
    const size_t n = (size_t)host_tallies[4];
    if (n) {   // the emitted entries alone
        FA_CUDA_TRY(H.back(n, pairs));
        FA_CUDA_TRY(H.sync());
    }
    *entry_count = (int32_t)n;
    for (int k = 0; counters && k < 4; ++k) counters[k] = host_tallies[k];
    return FA_OK;
}

int weight_resample(CallContext &C, const float *rows, long long row_count, int in_len, int out_len, float *out) {
    const cudaStream_t s = C.stream;
    const long long total = row_count * out_len;
    HostStaging H(true, s);
    const float *d_rows;
    float *d_out;
    const int st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        d_rows = l.in(rows, (size_t)(row_count * in_len));
        d_out = l.out(out, (size_t)total);
    });
    if (st != FA_OK) return st;
    const unsigned grid = (unsigned)std::min<long long>((total + kThreads - 1) / kThreads, 65535);
    FA_CUDA_TRY(launch(weight_resample_kernel, dim3(grid), dim3(kThreads), 0, s, d_rows, total, in_len, out_len, d_out));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

} // namespace prepare
} // namespace fa
