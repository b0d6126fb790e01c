// Diarizer timelines on the GPU (interface: timeline_plan.h; arithmetic: timeline_core.cuh).
//
//   timeline_scan_kernel       one warp per session, one lane per speaker: both passes of updateSegments, the
//                              segments into the lane's staging slot, the finalized-pass scratch kept; then the warp
//                              appends the finalized rows to the ring and replaces the tentative rows
//   timeline_pack_kernel       one CTA: an exclusive scan over the lanes' counts (call order, speaker-major), then the
//                              staged segments copied into the two compact output lists
//   timeline_finalize_kernel   one CTA per session holding tentative rows: those rows appended to the ring
//
// A push is two launches and a finalize at most one, whatever the session count.  Each lane's pass is sequential in
// time; it reads its column through a lane-private tile in shared memory, filled kTile rows at a time with independent
// loads, so the loads of a tile overlap instead of each step waiting for one.
#include "timeline_plan.h"

#include <algorithm>

namespace fa {
namespace timeline {

namespace {

constexpr int kWarps = 4;           // sessions per CTA of the scan
constexpr int kTile = 32;           // rows per lane prefetched into shared memory
constexpr int kPackThreads = 1024;

// Column `stride`-strided rows p[i * stride], i < n, through the lane's tile: element j of the tile at tile[j * 32].
struct TileRows {
    const float *p;
    long long n;
    int stride;
    float *tile;
    long long base;
    __device__ float operator()(long long i) {
        if (i >= base + kTile) {
            base = i;
#pragma unroll
            for (int j = 0; j < kTile; ++j) tile[j * 32] = i + j < n ? __ldg(p + (i + j) * stride) : 0.0f;
        }
        return tile[(i - base) * 32];
    }
};

__global__ void __launch_bounds__(kWarps * 32)
timeline_scan_kernel(Params c, Layout l, const PushJob *__restrict__ jobs, int count, const float *__restrict__ fin,
                     const float *__restrict__ ten, StoredScratch *__restrict__ scratch, float *__restrict__ rows,
                     Segment *__restrict__ stage, int *__restrict__ lane_counts, int lanes,
                     int64_t *__restrict__ fin_counts, int64_t *__restrict__ ten_counts) {
    __shared__ float tiles[kWarps][kTile * 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kWarps + warp;
    if (i >= count) return;   // warp-uniform
    const PushJob J = jobs[i];
    const int S = l.speakers;
    long long nf = 0, nt = 0;
    if (lane < S) {
        StoredScratch *sp = scratch + J.slot * S + lane;
        Scratch a = load_scratch(*sp);
        Segment *slot = stage + J.stage + lane * J.bound;
        auto emit = [&](const Segment &s, bool finalized) {
            slot[nf + nt] = s;
            if (finalized) ++nf;
            else ++nt;
        };
        float *tile = &tiles[warp][lane];
        TileRows fr{fin + J.fin + lane, J.n, S, tile, -(long long)kTile};
        TileRows tr{ten + J.ten + lane, J.m, S, tile, -(long long)kTile};
        push_lane(c, a, lane, J.cursor, J.n, fr, J.m, tr, emit);
        *sp = store_scratch(a);
        lane_counts[J.counts + lane] = (int)nf;
        lane_counts[lanes + J.counts + lane] = (int)nt;
    }
    long long sf = nf, st = nt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sf += __shfl_xor_sync(0xffffffffu, sf, o);
        st += __shfl_xor_sync(0xffffffffu, st, o);
    }
    if (lane == 0) {
        fin_counts[i] = sf;
        ten_counts[i] = st;
    }
    // the stored predictions: the last min(n, ring_rows) finalized rows at frame % ring_rows, then the tentative rows
    float *dst = rows + J.slot * l.slot_floats;
    if (l.ring_rows > 0) {
        const long long j0 = J.n > l.ring_rows ? J.n - l.ring_rows : 0;
        for (long long q = j0 * S + lane; q < J.n * S; q += 32) {
            const long long j = q / S;
            dst[((J.cursor + j) % l.ring_rows) * S + (q - j * S)] = fin[J.fin + q];
        }
    }
    float *tdst = dst + l.ring_rows * S;
    for (long long q = lane; q < J.m * S; q += 32) tdst[q] = ten[J.ten + q];
}

// Exclusive scan of one value per thread over the CTA (two lists at once).
__device__ void block_exclusive_scan(long long &a, long long &b, long long *warp_a, long long *warp_b) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long xa = __shfl_up_sync(0xffffffffu, ia, o), xb = __shfl_up_sync(0xffffffffu, ib, o);
        if (lane >= o) {
            ia += xa;
            ib += xb;
        }
    }
    if (lane == 31) {
        warp_a[warp] = ia;
        warp_b[warp] = ib;
    }
    __syncthreads();
    if (warp == 0) {
        long long wa = lane < (int)(blockDim.x >> 5) ? warp_a[lane] : 0, wb = lane < (int)(blockDim.x >> 5) ? warp_b[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long xa = __shfl_up_sync(0xffffffffu, wa, o), xb = __shfl_up_sync(0xffffffffu, wb, o);
            if (lane >= o) {
                wa += xa;
                wb += xb;
            }
        }
        warp_a[lane] = wa;
        warp_b[lane] = wb;
    }
    __syncthreads();
    const long long pa = warp ? warp_a[warp - 1] : 0, pb = warp ? warp_b[warp - 1] : 0;
    a = pa + ia - a;
    b = pb + ib - b;
}

__global__ void __launch_bounds__(kPackThreads)
timeline_pack_kernel(int S, int lanes, const PushJob *__restrict__ jobs, const Segment *__restrict__ stage,
                     const int *__restrict__ lane_counts, long long *__restrict__ offsets, Segment *__restrict__ fin_out,
                     Segment *__restrict__ ten_out) {
    __shared__ long long warp_a[32], warp_b[32];
    // each thread scans a contiguous run of lanes
    const int per = (lanes + kPackThreads - 1) / kPackThreads;
    const int e0 = min(lanes, (int)threadIdx.x * per), e1 = min(lanes, e0 + per);
    long long a = 0, b = 0;
    for (int e = e0; e < e1; ++e) {
        a += lane_counts[e];
        b += lane_counts[lanes + e];
    }
    block_exclusive_scan(a, b, warp_a, warp_b);
    for (int e = e0; e < e1; ++e) {
        offsets[e] = a;
        offsets[lanes + e] = b;
        a += lane_counts[e];
        b += lane_counts[lanes + e];
    }
    __syncthreads();
    // one warp per lane's slot
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int e = warp; e < lanes; e += kPackThreads / 32) {
        const int i = e / S, k = e - i * S;
        const PushJob &J = jobs[i];
        const Segment *src = stage + J.stage + k * J.bound;
        const int nf = lane_counts[e], nt = lane_counts[lanes + e];
        Segment *fo = fin_out + offsets[e], *to = ten_out + offsets[lanes + e];
        for (int j = lane; j < nf; j += 32) fo[j] = src[j];
        for (int j = lane; j < nt; j += 32) to[j] = src[nf + j];
    }
}

__global__ void timeline_finalize_kernel(Layout l, const FinalizeJob *__restrict__ jobs, float *__restrict__ rows) {
    const FinalizeJob J = jobs[blockIdx.x];
    const int S = l.speakers;
    float *dst = rows + J.slot * l.slot_floats;
    const float *src = dst + l.ring_rows * S;
    const long long j0 = J.m > l.ring_rows ? J.m - l.ring_rows : 0;
    for (long long q = j0 * S + threadIdx.x; q < J.m * S; q += blockDim.x) {
        const long long j = q / S;
        dst[((J.cursor + j) % l.ring_rows) * S + (q - j * S)] = src[q];
    }
}

} // namespace

int launch_push(const Config &c, const Layout &l, const PushJob *d_jobs, int count, const float *fin, const float *ten,
                StoredScratch *scratch, float *rows, Segment *stage, int *lane_counts, int64_t *fin_counts,
                int64_t *ten_counts, cudaStream_t s) {
    const int blocks = (count + kWarps - 1) / kWarps;
    FA_CUDA_TRY(launch(timeline_scan_kernel, dim3(blocks), dim3(kWarps * 32), 0, s, c.params(), l, d_jobs, count, fin, ten,
                       scratch, rows, stage, lane_counts, count * l.speakers, fin_counts, ten_counts));
    return FA_OK;
}

int launch_pack(const Layout &l, int lanes, const PushJob *d_jobs, const Segment *stage, const int *lane_counts,
                long long *lane_offsets, Segment *fin_out, Segment *ten_out, cudaStream_t s) {
    FA_CUDA_TRY(launch(timeline_pack_kernel, dim3(1), dim3(kPackThreads), 0, s, l.speakers, lanes, d_jobs, stage,
                       lane_counts, lane_offsets, fin_out, ten_out));
    return FA_OK;
}

int launch_finalize(const Layout &l, const FinalizeJob *d_jobs, int count, float *rows, cudaStream_t s) {
    FA_CUDA_TRY(launch(timeline_finalize_kernel, dim3(count), dim3(128), 0, s, l, d_jobs, rows));
    return FA_OK;
}

} // namespace timeline
} // namespace fa
