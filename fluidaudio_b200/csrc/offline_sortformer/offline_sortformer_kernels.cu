// Offline Sortformer windows on the GPU (offline_sortformer.h, offline_sortformer_core.cuh).  Kernels:
//   osf_model_inputs_kernel  runOffline's copy for every window of every file: a CTA transposes 32 frames x 128 mels
//                            of one window through shared memory, reading whole time-major rows and writing 128-byte
//                            runs of each channel; a tile past validMel writes its zeros without reading
//   osf_stitch_kernel        processComplete's stitching: one warp per file walks its windows in order.  Per window
//                            it stages the overlap rows of the timeline and the window in shared memory, 16 lanes run
//                            the correlation chains, 24 lanes score the permutations and a warp reduction picks the
//                            first best one; then the lanes write the window's rows through the inverse mapping.
#include "offline_sortformer.h"

#include <algorithm>
#include <cfloat>
#include <cstring>
#include <cuda_runtime.h>
#include <vector>

namespace fa {
namespace offline_sortformer {

namespace {

constexpr int kThreads = 256;
constexpr int kTileFrames = 32;
constexpr int kTiles = kWindowMel / kTileFrames;   // tiles per window
constexpr int kStitchWarps = 2;                    // files per stitch CTA
constexpr int kStage = (kWindowOut - 1) * kSpeakers;
constexpr unsigned kFull = 0xffffffffu;

struct WindowJob {
    long long src;   // the window's first mel row, as a float offset from the call's first file
    int valid_mel, pad;
};

struct FileJob {
    long long frames, row0, win0;   // mel frames, first output row, first window
    int windows, pad;
};

__global__ void __launch_bounds__(kThreads)
    osf_model_inputs_kernel(const WindowJob *__restrict__ jobs, const float *__restrict__ mel,
                            float *__restrict__ out, int32_t *__restrict__ mel_length) {
    __shared__ float tile[kTileFrames][kMels + 1];
    const long long w = blockIdx.x / kTiles;
    const int t0 = (int)(blockIdx.x % kTiles) * kTileFrames;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const WindowJob J = jobs[w];
    float *O = out + (size_t)w * kMels * kWindowMel + t0 + lane;
    if (t0 == 0 && threadIdx.x == 0) mel_length[w] = J.valid_mel;
    if (t0 >= J.valid_mel) {
        for (int c = warp; c < kMels; c += kThreads / 32) O[(size_t)c * kWindowMel] = 0.0f;
        return;
    }
    for (int r = warp; r < kTileFrames; r += kThreads / 32) {
        const bool valid = t0 + r < J.valid_mel;
        const float *row = mel + J.src + (long long)(t0 + r) * kMels + lane;
        for (int q = 0; q < kMels; q += 32) tile[r][q + lane] = valid ? row[q] : 0.0f;
    }
    __syncthreads();
    for (int c = warp; c < kMels; c += kThreads / 32) O[(size_t)c * kWindowMel] = tile[lane][c];
}

__global__ void __launch_bounds__(kStitchWarps * 32)
    osf_stitch_kernel(const FileJob *__restrict__ jobs, int count, int overlap, const float *__restrict__ preds,
                      float *__restrict__ out, int32_t *__restrict__ mappings) {
    __shared__ float stage[kStitchWarps][2][kStage];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kStitchWarps + warp;
    if (i >= count) return;
    const FileJob J = jobs[i];
    const long long total = total_out(J.frames);
    float *G = stage[warp][0], *Wn = stage[warp][1];
    float *O = out + J.row0 * kSpeakers;
    long long covered = 0;   // frames [0, covered) are filled: windows are contiguous, so coverage is a prefix
    for (int k = 0; k < J.windows; ++k) {
        const Window win = window_at(J.frames, overlap, k);
        const long long g_start = win.mel_start / kSubsampling;
        const float *P = preds + (size_t)(J.win0 + k) * kWindowOut * kSpeakers;
        int best = 0;   // identity
        const int ov = k > 0 && overlap > 0 ? overlap_frames(overlap, win.valid_out, total, g_start) : 0;
        if (ov > 0) {
            for (int e = lane; e < ov * kSpeakers; e += 32) {
                G[e] = O[g_start * kSpeakers + e];
                Wn[e] = P[e];
            }
            __syncwarp();
            const float c = lane < kSpeakers * kSpeakers ? correlation(G, Wn, ov, lane >> 2, lane & 3) : 0.0f;
            const int p = lane < kPerms ? lane : 0;
            float cg[kSpeakers];
            for (int g = 0; g < kSpeakers; ++g) cg[g] = __shfl_sync(kFull, c, g * kSpeakers + perm_at(p, g));
            float s = score(cg[0], cg[1], cg[2], cg[3]);
            // the first permutation, in enumeration order, whose score beats every earlier one and -FLT_MAX: the
            // lowest index among the largest values above -FLT_MAX, compared as values (+0 == -0, NaN never wins)
            int valid = lane < kPerms && s > -FLT_MAX, idx = lane;
            for (int m = 16; m; m >>= 1) {
                const float os = __shfl_xor_sync(kFull, s, m);
                const int oi = __shfl_xor_sync(kFull, idx, m), ovd = __shfl_xor_sync(kFull, valid, m);
                if (ovd && (!valid || os > s || (os == s && oi < idx))) s = os, idx = oi, valid = ovd;
            }
            best = valid ? idx : 0;
        }
        const int w = lane & 3;   // every element this lane writes is of window column w
        int m = 0;
        for (int g = 0; g < kSpeakers; ++g)
            if (perm_at(best, g) == w) m = g;
        if (mappings && lane < kSpeakers) mappings[(J.win0 + k) * kSpeakers + lane] = m;
        for (int e = lane; e < win.valid_out * kSpeakers; e += 32) {
            const long long gf = g_start + (e >> 2);
            if (gf >= total) break;
            float *dst = O + gf * kSpeakers + m;
            const float v = P[e];
            *dst = gf < covered ? average(*dst, v) : v;
        }
        const long long end = g_start + win.valid_out < total ? g_start + win.valid_out : total;
        covered = end > covered ? end : covered;
        __syncwarp();   // window k + 1 stages and averages the rows window k wrote
    }
}

template <typename Job> int upload_jobs(CallContext &C, const std::vector<Job> &jobs) {
    const size_t bytes = jobs.size() * sizeof(Job);
    int st = C.stage.reserve(bytes);
    if (st != FA_OK) return st;
    std::memcpy(C.stage.host.data(), jobs.data(), bytes);
    return C.stage.upload(bytes, C.stream);
}

} // namespace

int model_inputs(CallContext &C, int overlap, int count, const float *mel, const int64_t *mel_offsets,
                 const int64_t *mel_frames, long long windows, bool device, float *model_mel, int32_t *mel_length) {
    if (windows == 0) return FA_OK;
    long long lo = -1, hi = 0;   // the span of mel the files' rows lie in
    for (int i = 0; i < count; ++i) {
        if (mel_frames[i] == 0) continue;
        lo = lo < 0 ? mel_offsets[i] : std::min(lo, (long long)mel_offsets[i]);
        hi = std::max(hi, (long long)(mel_offsets[i] + mel_frames[i] * kMels));
    }
    std::vector<WindowJob> jobs((size_t)windows);
    size_t at = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = window_count(mel_frames[i], overlap);
        for (long long k = 0; k < n; ++k) {
            const Window w = window_at(mel_frames[i], overlap, k);
            jobs[at++] = WindowJob{mel_offsets[i] - lo + w.mel_start * kMels, w.valid_mel, 0};
        }
    }
    int st = upload_jobs(C, jobs);
    if (st != FA_OK) return st;
    HostStaging H(!device, C.stream);
    const float *k_mel;
    float *k_out;
    int32_t *k_len;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_mel = l.in(mel + lo, (size_t)(hi - lo));
        k_out = l.out(model_mel, (size_t)windows * kMels * kWindowMel);
        k_len = l.out(mel_length, (size_t)windows);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(osf_model_inputs_kernel, dim3((unsigned)(windows * kTiles)), kThreads, 0, C.stream,
                       static_cast<const WindowJob *>(C.stage.device.data()), k_mel, k_out, k_len));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

int stitch(CallContext &C, int overlap, int count, const int64_t *mel_frames, const float *speaker_preds,
           long long windows, long long rows, bool device, float *predictions, int32_t *mappings) {
    if (windows == 0) return FA_OK;
    std::vector<FileJob> jobs((size_t)count);
    long long row = 0, win = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = window_count(mel_frames[i], overlap);
        jobs[i] = FileJob{mel_frames[i], row, win, (int)n, 0};
        row += total_out(mel_frames[i]);
        win += n;
    }
    int st = upload_jobs(C, jobs);
    if (st != FA_OK) return st;
    HostStaging H(!device, C.stream);
    const float *k_preds;
    float *k_out;
    int32_t *k_map;
    st = H.carve(C.d_buf, [&](HostStaging::Layout &l) {
        k_preds = l.in(speaker_preds, (size_t)windows * kWindowOut * kSpeakers);
        k_out = l.out(predictions, (size_t)rows * kSpeakers);
        k_map = l.out(mappings, (size_t)windows * kSpeakers);
    });
    if (st != FA_OK) return st;
    FA_CUDA_TRY(launch(osf_stitch_kernel, dim3((unsigned)((count + kStitchWarps - 1) / kStitchWarps)),
                       kStitchWarps * 32, 0, C.stream, static_cast<const FileJob *>(C.stage.device.data()), count,
                       overlap, k_preds, k_out, k_map));
    FA_CUDA_TRY(H.finish());
    return FA_OK;
}

} // namespace offline_sortformer
} // namespace fa
