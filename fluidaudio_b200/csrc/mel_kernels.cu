// Fused log-mel frontend for sm_90a:  pre-emphasis -> Hann window -> 512-point real FFT -> |.|^2 ->
// Slaney mel filterbank -> log, one persistent CTA per SM.
//
// Re-implements Sources/FluidAudio/Shared/AudioMelSpectrogram.swift:325-456 (computeFlatTransposed),
// :185-292 (computeFlat) and :132-178 (compute) — the three differ only in (pad, window offset, pre-emphasis,
// output layout), which are kernel parameters here.
//
// Data flow per tile of kTileFrames (16) frames, two CTAs of 8 warps per SM so that one CTA's FP64 transform phase
// overlaps the other's float32 mel/log phase and barrier waits:
//   HBM --cp.async.bulk (TMA 1-D, mbarrier complete_tx)--> raw[2]   double-buffered, prefetched one tile ahead
//   raw --pre-emphasis--> ptile                                       all threads
//   ptile --one warp per frame: FFT256 + recombination--> power[32][257]
//   power --lane = frame, warp = mel: banded dot + log--> otile / HBM
// The transform runs in FP64 (see mel_core.cuh for why), everything the reference does in float32 stays float32.
// HBM traffic is the algorithmic minimum: every sample is read once (plus a 352-sample halo per tile) and
// every log-mel value is written once, both fully coalesced.
//
// The mel filterbank is applied as a BANDED contraction on the FP32 pipe, not as a tensor-core GEMM: each
// FFT bin feeds at most two triangular filters, so the dense [T x 257] x [257 x nMels] product is >97 % zeros
// (514 useful MACs per frame out of 20 560 at 80 mels), and bf16 operands cannot meet the 1e-4 log-mel parity
// bound (SURVEY.md §7 H3).  See DESIGN.md §4.
#include "mel_core.cuh"
#include "mel_plan.h"

#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>
#include <vector>

namespace fa {
namespace mel {

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// 1-D bulk copy global -> shared (TMA engine), completion signalled on an mbarrier.  SASS: UBLKCP.
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ kernel
struct TileGeom {
    int unit;          // index into units[]
    long long f0;      // first frame of the tile (absolute frame index inside the clip)
    int nf;            // frames in this tile (1..32)
    long long a0;      // audio index of ptile[0]  (= f0*hop - pad)
    long long base;    // audio index of raw[0]    (= floor4(a0 - 1), may be negative)
    long long gs, ge;  // bulk-copied audio range [gs, ge), both multiples of 4 (empty if ge <= gs)
};

__device__ __forceinline__ const MelUnit &unit_at(const MelLaunch &P, int idx) { return P.inline_unit ? P.unit0 : P.units[idx]; }

__device__ __forceinline__ TileGeom tile_geom(const MelLaunch &P, int tile) {
    // units are sorted by tile_begin; binary search for the unit that owns this tile
    int lo = 0, hi = P.inline_unit ? 0 : P.num_units - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (P.units[mid].tile_begin <= tile) lo = mid; else hi = mid - 1;
    }
    const MelUnit &u = P.inline_unit ? P.unit0 : P.units[lo];
    TileGeom g;
    g.unit = lo;
    g.f0 = u.frame_begin + (long long)kTileFrames * (tile - u.tile_begin);
    const long long rem = u.frame_begin + u.frame_count - g.f0;
    g.nf = rem < kTileFrames ? (int)rem : kTileFrames;
    g.a0 = g.f0 * P.hop - P.pad;
    const long long need0 = g.a0 - 1;
    g.base = (need0 >= 0) ? (need0 & ~3LL) : -(((-need0) + 3) & ~3LL);
    long long ge = (g.a0 + P.pt_len + 3) & ~3LL;
    const long long n4 = u.n & ~3LL;
    if (ge > n4) ge = n4;
    g.gs = g.base < 0 ? 0 : g.base;
    g.ge = ge;
    if (!P.use_tma) g.ge = g.gs;   // nothing is bulk-copied: every sample comes through the read-only path
    return g;
}

// Geometry + the unit fields a tile needs, computed ONCE per tile by thread 0 and broadcast through shared memory (three
// rotating slots): every thread recomputing it (binary search, 64-bit index math, a 56-byte struct copy) three times per
// tile was 6 % of the kernel's instructions (profiles/r02_mel.md).
struct TileInfo {
    TileGeom g;
    long long audio_off, n, out_off, out_stride;
    float last;
    int pad_;
};
__device__ __forceinline__ void make_tile_info(const MelLaunch &P, int tile, TileInfo &ti) {
    ti.g = tile_geom(P, tile);
    const MelUnit &u = unit_at(P, ti.g.unit);
    ti.audio_off = u.audio_off;
    ti.n = u.n;
    ti.out_off = u.out_off;
    ti.out_stride = u.out_stride;
    ti.last = u.last;
}

template <int kWarps, typename V, int kLayout>   // kLayout: 0 time-major [T x nMels], 1 mel-major [nMels x stride]
__global__ void __launch_bounds__(kWarps * 32, 2) mel512_kernel(const MelLaunch P) {
    constexpr int kF = vtraits<V>::kFrames;   // frames one warp transforms together (2: packed float32 pairs)
    extern __shared__ __align__(128) unsigned char smem[];
    float *raw0 = reinterpret_cast<float *>(smem);
    float *raw1 = raw0 + P.raw_cap;
    float *ptile = raw1 + P.raw_cap;
    cpxv<V> *fftbuf = reinterpret_cast<cpxv<V> *>(ptile + P.pt_cap);   // kWarps * kFftPad complex values (16 bytes each)
    float *power = reinterpret_cast<float *>(fftbuf + kWarps * kFftPad);   // (kTileFrames / 2) pair rows x kPairStride
    float *otile = power + (kTileFrames / 2) * kPairStride;  // kTileFrames rows of ot_stride floats
    const int ot_stride = P.ot_stride;                       // n_mels + 4 (rows stay 16-byte aligned) or n_mels + 1
    float *fbw = otile + kTileFrames * ot_stride;            // fb_nnz_cap
    int4 *fbmeta = reinterpret_cast<int4 *>(fbw + P.fb_cap);   // n_slots x {first bin, quads, weight offset, mel bin or -1}
    uint64_t *bars = reinterpret_cast<uint64_t *>(fbmeta + P.n_slots);
    TileInfo *tinfo = reinterpret_cast<TileInfo *>(bars + 2);   // [3]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < P.fb_nnz; i += kWarps * 32) fbw[i] = P.fb_w[i];
    for (int i = tid; i < P.n_slots; i += kWarps * 32) fbmeta[i] = P.fb_slots[i];
    for (int i = tid; i < (kTileFrames / 2) * kPairStride; i += kWarps * 32) power[i] = 0.0f;   // rows of partial tiles, pad columns
    // per-lane constants (window slots, twiddles, butterfly addresses): built on the host once per plan (FP64 sin / cos
    // inlined here cost ~3 % of the kernel and 9 000 SASS lines), one struct copy per thread
    const LaneTables<V> T = reinterpret_cast<const LaneTables<V> *>(P.lane_tab)[lane];
    __syncthreads();

    cpxv<V> *buf = fftbuf + warp * kFftPad;

    auto issue = [&](int tile, int buf, TileInfo &slot) {   // thread 0 only: publishes the tile's info, starts its bulk copy
        make_tile_info(P, tile, slot);
        const TileGeom &g = slot.g;
        float *dst = buf ? raw1 : raw0;
        if (g.ge > g.gs) {
            const uint32_t bytes = (uint32_t)((g.ge - g.gs) * 4);
            mbar_expect_tx(&bars[buf], bytes);
            bulk_g2s(dst + (g.gs - g.base), P.audio + slot.audio_off + g.gs, bytes, &bars[buf]);
        } else {
            mbar_arrive(&bars[buf]);
        }
    };

    // pre-emphasis of one tile from its raw buffer into ptile (zero outside [0, n))
    auto preemphasize = [&](const TileInfo &u, const float *raw) {   // u.n / u.last / u.audio_off: the owning clip
        const TileGeom &g = u.g;
        const float a = P.preemph;
        const bool interior = g.a0 >= 1 && g.a0 - 1 >= g.gs && g.a0 + P.pt_len <= g.ge && g.a0 + P.pt_len <= u.n;
        if (interior) {
            // every sample of the tile and its predecessor came through the bulk copy (conflict-free, unit stride)
            const float *src = raw + (g.a0 - g.base);   // src[t] = x(a0 + t), src[-1] valid
            if (((g.a0 - g.base) & 3) == 0 && (P.pt_len & 3) == 0) {   // 16-byte aligned rows: four samples per step
                const float4 *s4 = reinterpret_cast<const float4 *>(src);
                float4 *d4 = reinterpret_cast<float4 *>(ptile);
                for (int q = tid; q < (P.pt_len >> 2); q += kWarps * 32) {
                    const float4 x = s4[q];
                    float4 y = x;
                    const float prev = src[4 * q - 1];   // (a shuffle from the neighbour lane saves 4 wavefronts per frame but costs
                                                         //  more instructions than it saves: measured 0.3135 vs 0.3096 ms)
                    if (a != 0.0f) {
                        y.x = preemph_rest(x.x, prev, a);
                        y.y = preemph_rest(x.y, x.x, a);
                        y.z = preemph_rest(x.z, x.y, a);
                        y.w = preemph_rest(x.w, x.z, a);
                    }
                    d4[q] = y;
                }
            } else if (a == 0.0f) {
                for (int t = tid; t < P.pt_len; t += kWarps * 32) ptile[t] = src[t];
            } else {
                for (int t = tid; t < P.pt_len; t += kWarps * 32) ptile[t] = preemph_rest(src[t], src[t - 1], a);
            }
        } else {
            const float *gaudio = P.audio + u.audio_off;
            auto sample = [&](long long i) -> float {   // x(i) for -1 <= i < n
                if (i >= g.gs && i < g.ge) return raw[i - g.base];
                if (i < 0) return u.last;
                return __ldg(gaudio + i);
            };
            for (int t = tid; t < P.pt_len; t += kWarps * 32) {
                const long long i = g.a0 + t;
                float v = 0.0f;
                if (i >= 0 && i < u.n) {
                    const float x = sample(i);
                    if (a == 0.0f) v = x;
                    else if (i == 0) v = preemph_first(x, u.last, a);
                    else v = preemph_rest(x, sample(i - 1), a);
                }
                ptile[t] = v;
            }
        }
    };
    // time-major tile is contiguous in HBM: nf rows of n_mels floats; flat, fully coalesced copy out of otile
    auto copy_out = [&](float *dst, int total) {
        if (P.out_vec4) {   // rows are whole float4s and dst is 16-byte aligned (out, out_off checked by launch(); f0 % 16 == 0)
            float4 *d4 = reinterpret_cast<float4 *>(dst);
            for (int q = tid; q < (total >> 2); q += kWarps * 32) {
                const int e = 4 * q;
                const int row = (int)__umulhi((unsigned)e, P.inv_n_mels);                  // e / n_mels
                d4[q] = *reinterpret_cast<const float4 *>(otile + e + 4 * row);             // row stride n_mels + 4: one LDS.128
            }
        } else {   // any 4-byte aligned dst
            const int row_pad = ot_stride - P.n_mels;   // 4 or 1
            for (int idx = tid; idx < total; idx += kWarps * 32) {
                // idx / n_mels (exact for idx < 2^16); one mel: 2^32 does not fit inv_n_mels
                const int fi = P.n_mels == 1 ? idx : (int)__umulhi((unsigned)idx, P.inv_n_mels);
                dst[idx] = otile[idx + fi * row_pad];
            }
        }
    };

    // Software pipeline over the CTA's tiles, two block barriers per tile:
    //   phase A(i): copy-out of tile i-1 (otile -> HBM)  +  FFT of tile i (ptile -> power)
    //   phase B(i): mel + log of tile i (power -> otile)  +  pre-emphasis of tile i+1 (raw -> ptile), TMA for tile i+2
    // The bulk copy of a tile is issued two phases B ahead of its use, its raw buffer was last read one phase B earlier.
    const int first = blockIdx.x, stride = gridDim.x;
    if (first >= P.total_tiles) return;
    if (tid == 0) {
        issue(first, 0, tinfo[0]);
        if (first + stride < P.total_tiles) issue(first + stride, 1, tinfo[1]);
    }
    __syncthreads();
    mbar_wait(&bars[0], 0);
    preemphasize(tinfo[0], raw0);
    __syncthreads();
    float *pending_dst = nullptr;
    int pending_total = 0;
    int it = 0, slot = 0;   // slot = it % 3
    for (int tile = first; tile < P.total_tiles; tile += stride, ++it, slot = slot == 2 ? 0 : slot + 1) {
        const TileInfo &u = tinfo[slot];
        const int nf = u.g.nf;

        // ---- phase A: previous tile's copy-out, then one warp per frame (pair): FFT256 + recombination + power ----
        if (pending_dst) copy_out(pending_dst, pending_total);
        for (int fi = warp * kF; fi < nf; fi += kWarps * kF) {   // kF == 2: frames fi and fi + 1 (kTileFrames is even)
            const float *pf = ptile + fi * P.hop;
            V re[8], im[8];
            if (P.mid_full) pass1<true>(lane, pf, P.hop, T, buf); else pass1<false>(lane, pf, P.hop, T, buf);
            __syncwarp();
            pass2_load(lane, buf, re, im);
            __syncwarp();
            pass2_store(lane, T, re, im, buf);
            __syncwarp();
            pass3_post(lane, buf, T, power + (fi >> 1) * kPairStride + (fi & 1));   // pair row (+ slot on the FP64 path)
            __syncwarp();
        }
        __syncthreads();

        // ---- phase B: mel filterbank + log; a warp covers kTileFrames frames x (32 / kTileFrames) mel bins -------
        const int next = tile + stride;
        const int slot1 = slot == 2 ? 0 : slot + 1, slot2 = slot1 == 2 ? 0 : slot1 + 1;
        if (tid == 0 && next + stride < P.total_tiles) {
            fence_proxy_async();   // generic-proxy reads of this raw buffer (pre-emphasis, previous phase B) precede the async write
            issue(next + stride, it & 1, tinfo[slot2]);   // slot2 held tile it-1: nobody reads it any more
        }
        {
            constexpr int kPairs = kTileFrames / 2, kGroup = 32 / kPairs;   // lane = (frame pair, one of kGroup mel bins)
            const int pl = lane % kPairs, mg = lane / kPairs;
            const float *prow = power + pl * kPairStride;
            float *orow = otile + (2 * pl) * ot_stride;
            float *gout = kLayout == 1 ? P.out + u.out_off + u.g.f0 + 2 * pl : nullptr;   // mel-major: this pair's columns
            // slots, not mel bins: the plan deals the groups of four filters to the warps by band width (LPT), so that the
            // warp with the widest (highest) filters does not hold the block barrier; md.w = the slot's mel bin, -1 = empty
            for (int slot = warp * kGroup + mg; slot < P.n_slots; slot += kWarps * kGroup) {
                const int4 md = fbmeta[slot];
                // two frames per lane; rows beyond the tile's last frame hold finite leftovers: computed and
                // dropped, no divergent branch
                const float2 a2 = mel_dot_pairs(reinterpret_cast<const float4 *>(prow + 2 * md.x),
                                                reinterpret_cast<const float4 *>(fbw + md.z), md.y);
                const float v0 = log_value(a2.x, P.log_floor, P.log_clamped, P.log_normal),
                            v1 = log_value(a2.y, P.log_floor, P.log_clamped, P.log_normal);
                const int m = md.w;
                if (m < 0) continue;
                if (kLayout == 0) {
                    orow[m] = v0;
                    orow[ot_stride + m] = v1;
                } else {
                    float *g = gout + (long long)m * u.out_stride;
                    if (2 * pl < nf) g[0] = v0;
                    if (2 * pl + 1 < nf) g[1] = v1;
                }
            }
        }
        if (kLayout == 0) {
            pending_dst = P.out + u.out_off + u.g.f0 * P.n_mels;
            pending_total = nf * P.n_mels;
        }
        if (next < P.total_tiles) {
            const int nb = (it + 1) & 1;
            mbar_wait(&bars[nb], (uint32_t)((it + 1) >> 1) & 1u);
            preemphasize(tinfo[slot1], nb ? raw1 : raw0);
        }
        __syncthreads();
    }
    if (pending_dst) copy_out(pending_dst, pending_total);
}


// ------------------------------------------------------------------------------------------------ any-nFFT kernel
// AudioMelSpectrogram is parametric (AudioMelSpectrogram.swift:59-70) and LS-EEND derives nFFT = nextPow2(winLength)
// (Diarizer/LS-EEND/LSEENDTypes.swift:55-57): nFFT other than 512, or an odd hop, take this kernel.  Same contract, same
// unit / tile bookkeeping and the same packed filterbank as mel512_kernel; one warp per frame, the transform an FP64
// radix-2 decimation-in-time FFT of the real frame in shared memory (twiddles from an FP64 table), power rounded once
// to float32.  A correctness-first path: ~6x the instructions per frame of the specialised kernel.
// The torch-style frontends (fa_mel_create_ex) also run here, as three compile-time variants; <false, kSpecPower, false>
// is AudioMelSpectrogram's kernel:
//   kReflect   .center reads reflect_index(i, n) (mel_core.cuh) instead of zeros outside the clip; no pre-emphasis;
//   kSpectrum  kSpecPower: the tile holds 4|X|^2 and the weights 1/4 of the table; kSpecMagnitude: sqrt of the float32
//              power (rounded once from the FP64 transform), kSpecGeneral: powf(|X|, p); both with unscaled weights;
//   kAffine    out = (log - log_mean) / log_std, two rounded float32 operations as the Swift states them.
struct GenericParams {
    int n_fft, log2n, bins, prow;      // prow: floats per power row (bins rounded up to quads + 4)
    const cpxd *tw;                    // W_n^k, k < n/2
    int warps;
    float spectrum_power;              // kSpecGeneral: p
    float log_mean, log_std;           // kAffine
};

template <bool kReflect, int kSpectrum, bool kAffine>
__global__ void __launch_bounds__(256) mel_generic_kernel(const MelLaunch P, const GenericParams G) {
    extern __shared__ __align__(16) unsigned char smem[];
    cpxd *tw = reinterpret_cast<cpxd *>(smem);                                   // n/2
    cpxd *fft = tw + G.n_fft / 2;                                                // warps x n
    float *power = reinterpret_cast<float *>(fft + (size_t)G.warps * G.n_fft);   // warps x prow
    float *win = power + (size_t)G.warps * G.prow;                               // n (0 outside the window)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = G.warps * 32;
    for (int i = tid; i < G.n_fft / 2; i += nthreads) tw[i] = G.tw[i];
    for (int i = tid; i < G.n_fft; i += nthreads) win[i] = P.in_tab[i] ? P.win_tab[i] : 0.0f;
    for (int i = tid; i < G.warps * G.prow; i += nthreads) power[i] = 0.0f;
    __syncthreads();
    cpxd *buf = fft + (size_t)warp * G.n_fft;
    float *prow = power + (size_t)warp * G.prow;
    const float a = P.preemph;
    for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
        const TileGeom g = tile_geom(P, tile);
        const MelUnit u = unit_at(P, g.unit);
        const float *x = P.audio + u.audio_off;
        for (int fi = warp; fi < g.nf; fi += G.warps) {
            const long long f = g.f0 + fi;
            const long long base = f * P.hop - P.pad;
            // pre-emphasis + window into bit-reversed order
            for (int j = lane; j < G.n_fft; j += 32) {
                const long long i = base + j;
                float v = 0.0f;
                if (kReflect) {
                    if (u.n > 0 && P.in_tab[j]) v = __fmul_rn(__ldg(x + reflect_index(i, u.n)), win[j]);
                } else if (i >= 0 && i < u.n && P.in_tab[j]) {
                    const float xi = __ldg(x + i);
                    if (a == 0.0f) v = xi;
                    else if (i == 0) v = preemph_first(xi, u.last, a);
                    else v = preemph_rest(xi, __ldg(x + i - 1), a);
                    v = __fmul_rn(v, win[j]);
                }
                cpxd z;
                z.x = (double)v;
                z.y = 0.0;
                buf[__brev((unsigned)j) >> (32 - G.log2n)] = z;
            }
            __syncwarp();
            for (int s = 0; s < G.log2n; ++s) {
                const int half = 1 << s, step = G.n_fft >> (s + 1);
                for (int t = lane; t < G.n_fft / 2; t += 32) {
                    const int j = t & (half - 1);
                    const int ia = ((t >> s) << (s + 1)) + j, ib = ia + half;
                    const cpxd w = tw[j * step], zb = buf[ib], za = buf[ia];
                    const double tr = zb.x * w.x - zb.y * w.y, ti = zb.x * w.y + zb.y * w.x;
                    cpxd o;
                    o.x = za.x - tr;
                    o.y = za.y - ti;
                    buf[ib] = o;
                    o.x = za.x + tr;
                    o.y = za.y + ti;
                    buf[ia] = o;
                }
                __syncwarp();
            }
            for (int b = lane; b < G.bins; b += 32) {
                const float xr = (float)buf[b].x, xi = (float)buf[b].y;
                const float pw = __fadd_rn(__fmul_rn(xr, xr), __fmul_rn(xi, xi));
                if (kSpectrum == kSpecPower) prow[b] = 4.0f * pw;   // the packed weights carry 1/4
                else if (kSpectrum == kSpecMagnitude) prow[b] = __fsqrt_rn(pw);
                else prow[b] = powf(__fsqrt_rn(pw), G.spectrum_power);   // CohereMelSpectrogram's pow(mag, magPower)
            }
            __syncwarp();
            for (int m = lane; m < P.n_mels; m += 32) {
                const int lo = P.fb_lo[m], nq = (P.fb_hi[m] - lo) >> 2;
                float v = log_value(mel_dot_quads(reinterpret_cast<const float4 *>(prow + lo),
                                                  reinterpret_cast<const float4 *>(P.fb_w + P.fb_off[m]), nq),
                                    P.log_floor, P.log_clamped);
                if (kAffine) v = __fdiv_rn(__fsub_rn(v, G.log_mean), G.log_std);
                if (P.layout == 0) P.out[u.out_off + f * P.n_mels + m] = v;
                else P.out[u.out_off + (long long)m * u.out_stride + f] = v;
            }
            __syncwarp();
        }
    }
}

// ------------------------------------------------------------------------------------------------ host plan
static constexpr int kCtasPerSm = 2;

// the specialised kernel's variant for a precision and a layout
typedef void (*Mel512Kernel)(const MelLaunch);
template <typename V> static Mel512Kernel mel512_variant(int layout) {
    return layout == FA_MEL_TIME_MAJOR ? mel512_kernel<kWarpsPerCta, V, FA_MEL_TIME_MAJOR>
                                       : mel512_kernel<kWarpsPerCta, V, FA_MEL_MEL_MAJOR>;
}
static Mel512Kernel mel512_variant(int precision, int layout) {
    return precision == FA_MEL_PRECISION_F64 ? mel512_variant<double>(layout) : mel512_variant<f32x2>(layout);
}

// the any-nFFT kernel's variant for a launch (see mel_generic_kernel)
typedef void (*GenericKernel)(const MelLaunch, const GenericParams);
template <bool R, int S> static GenericKernel generic_variant(bool affine) {
    return affine ? mel_generic_kernel<R, S, true> : mel_generic_kernel<R, S, false>;
}
template <bool R> static GenericKernel generic_variant(int spectrum, bool affine) {
    return spectrum == kSpecPower ? generic_variant<R, kSpecPower>(affine)
                                  : (spectrum == kSpecMagnitude ? generic_variant<R, kSpecMagnitude>(affine)
                                                                : generic_variant<R, kSpecGeneral>(affine));
}
static GenericKernel generic_variant(bool reflect, int spectrum, bool affine) {
    return reflect ? generic_variant<true>(spectrum, affine) : generic_variant<false>(spectrum, affine);
}

// Window placement of a mode (index of d_win_tab_mode / d_in_tab_mode / d_lane_tab): 0 centred at (nFFT - win) / 2,
// 1 at offset 0 for the legacy compute()
static int placement_of(int mode) { return mode == FA_MEL_LEGACY_COMPUTE ? 1 : 0; }
static int window_offset(const MelConfig &c, int placement) { return placement == 1 ? 0 : (c.n_fft - c.win_length) / 2; }

static_assert(sizeof(MelSlot) == sizeof(int4) && offsetof(MelSlot, mel) == offsetof(int4, w), "MelSlot is an int4");

// Device copy of a host table (at least one element, so that an empty table still has an address), complete on return:
// `v` may be a temporary, and the kernels that read the table run on `stream`.
template <typename T, typename U>
static int upload_table(DeviceBuffer<T> &b, const std::vector<U> &v, cudaStream_t stream) {
    const int st = b.grow(std::max<size_t>(1, v.size()) * sizeof(U));
    if (st != FA_OK) return st;
    if (v.empty()) return FA_OK;
    FA_CUDA_TRY(cudaMemcpyAsync(b.data(), v.data(), v.size() * sizeof(U), cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaStreamSynchronize(stream));
    return FA_OK;
}

int MelPlan::init(const MelConfig &c) {
    cfg = c;
    if (cfg.pad_to < 1) cfg.pad_to = 1;   // AudioMelSpectrogram.swift:72
    if (cfg.n_mels <= 0 || cfg.hop_length <= 0 || cfg.win_length <= 0 || cfg.n_fft <= 0 || cfg.sample_rate <= 0) {
        fa::set_error("mel config: all sizes must be positive");
        return FA_INVALID_ARGUMENT;
    }
    const bool pow2 = cfg.n_fft >= 32 && cfg.n_fft <= 4096 && (cfg.n_fft & (cfg.n_fft - 1)) == 0;
    if (!pow2 || cfg.win_length > cfg.n_fft || cfg.n_mels > 512 || cfg.hop_length > 65536) {
        fa::set_error("mel config unsupported by the sm_90a kernels: need nFFT a power of two in 32..4096, win <= nFFT, "
                      "nMels <= 512 (got nFFT=%d hop=%d win=%d nMels=%d)",
                      cfg.n_fft, cfg.hop_length, cfg.win_length, cfg.n_mels);
        return FA_UNSUPPORTED;
    }
    if (const char *why = check_ex_config(cfg)) {
        fa::set_error("mel ex config: %s", why);
        return FA_INVALID_ARGUMENT;
    }
    // the specialised kernel covers every in-repo caller's shape; anything else takes mel_generic_kernel, and so do
    // reflect padding, a spectrum other than |X|^2 and the affine epilogue (mel512_kernel only ever sees another table)
    const int spectrum = spectrum_kind(cfg.spectrum_power);
    generic = cfg.n_fft != kNfft || (cfg.hop_length & 1) || cfg.hop_length > 1024 || cfg.reflect() ||
              spectrum != kSpecPower || cfg.affine();
    const int n_fft = cfg.n_fft, bins = n_fft / 2 + 1;
    build_tables(cfg, window, filterbank);
    const MelBands bands = pack_bands(filterbank, cfg.n_mels, bins);
    fb_nnz = bands.nnz;
    n_slots = (int)bands.slots.size();

    int dev = 0;
    FA_CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    int st = sm90_device_props(dev, prop);
    if (st != FA_OK) return st;
    num_sms = prop.multiProcessorCount;

    if (!generic) {
        pt_len = (kTileFrames - 1) * cfg.hop_length + kNfft;
        pt_cap = (pt_len + 31) & ~31;
        raw_cap = (pt_len + 1 + 3 + 3 + 31) & ~31;   // whole 128-byte lines: the pre-emphasised tile behind it stays line-aligned
        fb_cap = (fb_nnz + 3) & ~3;
        smem_bytes = sizeof(float) * ((size_t)2 * raw_cap + pt_cap + 0 +
                                      (size_t)(kTileFrames / 2) * kPairStride + (size_t)kTileFrames * (cfg.n_mels + 4) + fb_cap) +
                     sizeof(cpxd) * (size_t)kWarpsPerCta * kFftPad + sizeof(int) * 4 * (size_t)n_slots + 8 +
                     2 * sizeof(uint64_t) + 3 * sizeof(TileInfo) + 16;
        // three tiles of 15 hops + 512 samples: past the opt-in limit (on H100 even hops from about 900 at 80 mels) the
        // any-nFFT kernel, whose budget does not depend on the hop, takes the configuration
        if (smem_bytes > (size_t)prop.sharedMemPerBlockOptin) {
            generic = true;
            pt_len = pt_cap = raw_cap = fb_cap = 0;
        }
    }

    for (auto &s : streams)
        if (st == FA_OK) st = s.create();
    if (st != FA_OK) return st;
    std::vector<float> win_tab;
    std::vector<uint8_t> in_tab;
    for (int pl = 0; pl < 2; ++pl) {
        place_window(window, n_fft, window_offset(cfg, pl), win_tab, in_tab);
        st = upload_table(d_win_tab_mode[pl], win_tab, streams[1]);
        if (st == FA_OK) st = upload_table(d_in_tab_mode[pl], in_tab, streams[1]);
        if (st != FA_OK) return st;
        if (!generic) {
            std::vector<LaneTables<double>> t64(32);
            std::vector<LaneTables<f32x2>> t32(32);
            for (int l = 0; l < 32; ++l) {
                load_lane_tables(l, win_tab.data(), in_tab.data(), t64[l]);
                load_lane_tables(l, win_tab.data(), in_tab.data(), t32[l]);
            }
            st = upload_table(d_lane_tab[pl][FA_MEL_PRECISION_F64], t64, streams[1]);
            if (st == FA_OK) st = upload_table(d_lane_tab[pl][FA_MEL_PRECISION_F32], t32, streams[1]);
            if (st != FA_OK) return st;
        }
    }
    // mel512_kernel finds the bins of a quad swizzled in its power tile, the any-nFFT kernel in natural order; the
    // weights carry 1/4 where the tile holds 4|X|^2
    st = upload_table(d_fb_w, pack_weights(filterbank, bands, bins, !generic, spectrum == kSpecPower ? 0.25f : 1.0f),
                      streams[1]);
    if (st == FA_OK) st = upload_table(d_fb_slots, bands.slots, streams[1]);
    if (st == FA_OK) st = upload_table(d_fb_lo, bands.lo, streams[1]);
    if (st == FA_OK) st = upload_table(d_fb_hi, bands.hi, streams[1]);
    if (st == FA_OK) st = upload_table(d_fb_off, bands.off, streams[1]);
    if (st != FA_OK) return st;
    if (generic) {
        // FP64 twiddle table W_n^k and the shared-memory budget: as many warps per CTA as fit beside it
        std::vector<cpxd> tw(n_fft / 2);
        for (int k = 0; k < n_fft / 2; ++k) tw[k] = unit_root(k, n_fft);
        st = upload_table(d_generic_tw, tw, streams[1]);
        if (st != FA_OK) return st;
        generic_prow = ((bins + 3) & ~3) + 4;
        int log2n = 0;
        while ((1 << log2n) < n_fft) ++log2n;
        generic_log2n = log2n;
        const size_t fixed = (size_t)(n_fft / 2) * sizeof(cpxd) + (size_t)n_fft * sizeof(float);
        const size_t per_warp = (size_t)n_fft * sizeof(cpxd) + (size_t)generic_prow * sizeof(float);
        generic_warps = (int)std::min<size_t>(8, ((size_t)prop.sharedMemPerBlockOptin - fixed - 1024) / per_warp);
        if (generic_warps < 1) {
            fa::set_error("mel config: nFFT %d does not fit shared memory", n_fft);
            return FA_UNSUPPORTED;
        }
        smem_bytes = fixed + per_warp * generic_warps;
        // the variants this handle launches: .center (reflected or not) and the other modes, which never reflect
        for (const bool r : {false, cfg.reflect()})
            FA_CUDA_TRY(cudaFuncSetAttribute(generic_variant(r, spectrum, cfg.affine()),
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
        return FA_OK;
    }
    for (const int precision : {FA_MEL_PRECISION_F64, FA_MEL_PRECISION_F32})
        for (const int layout : {FA_MEL_TIME_MAJOR, FA_MEL_MEL_MAJOR})
            FA_CUDA_TRY(cudaFuncSetAttribute(mel512_variant(precision, layout), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem_bytes));
    return FA_OK;
}

long long MelPlan::frame_count(long long n, int mode, long long expected) const {
    long long computed;   // C++ integer division truncates toward zero exactly like Swift's Int '/'
    if (mode == FA_MEL_PAD_CENTER) computed = 1 + (n + 2 * (long long)(cfg.n_fft / 2) - cfg.win_length) / cfg.hop_length;
    else if (mode == FA_MEL_PAD_PREPADDED) computed = std::max<long long>(0, (n - cfg.n_fft) / cfg.hop_length + 1);
    else computed = 1 + (n - cfg.win_length) / cfg.hop_length;
    return expected >= 0 ? expected : computed;
}

int MelPlan::ensure_events(size_t count) {
    while (events.size() < count) {
        Event e;
        const int st = e.create(cudaEventDisableTiming);
        if (st != FA_OK) return st;
        events.push_back(std::move(e));
    }
    return FA_OK;
}

static int tiles_of(long long frames) { return (int)((frames + kTileFrames - 1) / kTileFrames); }

int number_tiles(MelUnit *u, int count) {
    int tiles = 0;
    for (int i = 0; i < count; ++i) {
        u[i].tile_begin = tiles;
        tiles += tiles_of(u[i].frame_count);
    }
    return tiles;
}

int MelPlan::launch(const MelUnit *d_u, const MelUnit *h_u, int count, bool inline_unit, const float *d_audio_base,
                    float *d_out_base, int mode, int layout, cudaStream_t stream) {
    const int total_tiles = count > 0 ? h_u[count - 1].tile_begin + tiles_of(h_u[count - 1].frame_count) : 0;
    if (total_tiles <= 0) return FA_OK;
    MelLaunch P{};
    P.audio = d_audio_base;
    P.out = d_out_base;
    P.units = d_u;
    P.num_units = count;
    P.inline_unit = (inline_unit && count == 1) ? 1 : 0;
    if (P.inline_unit) P.unit0 = h_u[0];
    P.total_tiles = total_tiles;
    P.hop = cfg.hop_length;
    P.pad = mode == FA_MEL_PAD_CENTER ? cfg.n_fft / 2 : 0;
    P.preemph = mode == FA_MEL_LEGACY_COMPUTE ? 0.0f : cfg.preemph;
    P.n_mels = cfg.n_mels;
    P.log_floor = cfg.log_floor;
    P.log_clamped = cfg.log_floor_mode;
    P.ot_stride = (cfg.n_mels & 3) == 0 ? cfg.n_mels + 4 : cfg.n_mels + 1;
    // float4 copy-out only when every destination row is 16-byte aligned: the caller's d_out, a batch's out_offsets or a
    // pinned output may sit at any 4-byte boundary (h_u mirrors the launch's units)
    P.out_vec4 = (cfg.n_mels & 3) == 0 && (reinterpret_cast<uintptr_t>(d_out_base) & 15) == 0;
    for (int i = 0; i < count && P.out_vec4; ++i) P.out_vec4 = (h_u[i].out_off & 3) == 0;
    P.log_normal = cfg.log_floor >= 1e-37f ? 1 : 0;   // mel energies are >= 0: log's argument is then never a denormal
    P.layout = layout;
    const int pl = placement_of(mode);
    P.lane_tab = d_lane_tab[pl][precision == FA_MEL_PRECISION_F32 ? 1 : 0].data();
    P.win_tab = d_win_tab_mode[pl].data();
    P.in_tab = d_in_tab_mode[pl].data();
    P.fb_w = d_fb_w.data();
    P.fb_slots = d_fb_slots.data();
    P.n_slots = n_slots;
    P.fb_lo = d_fb_lo.data();
    P.fb_hi = d_fb_hi.data();
    P.fb_off = d_fb_off.data();
    P.fb_nnz = fb_nnz;
    P.fb_cap = fb_cap;
    P.pt_len = pt_len;
    P.pt_cap = pt_cap;
    P.raw_cap = raw_cap;
    // the bulk copy moves whole 16-byte runs of a unit's samples (tile_geom): the audio base must be 16-byte aligned and
    // every unit must start at a multiple of four floats, or every sample takes the read-only path
    P.use_tma = (reinterpret_cast<uintptr_t>(d_audio_base) & 15) == 0;
    for (int i = 0; i < count && P.use_tma; ++i) P.use_tma = (h_u[i].audio_off & 3) == 0;
    {
        const int off_w = window_offset(cfg, pl);
        P.mid_full = (off_w <= 64 && off_w + cfg.win_length >= 448) ? 1 : 0;
    }
    P.inv_n_mels = (unsigned)((0x100000000ull + (unsigned)cfg.n_mels - 1) / (unsigned)cfg.n_mels);
    if (generic) {
        GenericParams G{cfg.n_fft, generic_log2n, cfg.n_fft / 2 + 1, generic_prow,
                        static_cast<const cpxd *>(d_generic_tw.data()), generic_warps, cfg.spectrum_power, cfg.log_mean,
                        cfg.log_std};
        const int ggrid = std::min(total_tiles, num_sms * std::max(1, 16 / generic_warps));
        const GenericKernel kernel = generic_variant(mode == FA_MEL_PAD_CENTER && cfg.reflect(),
                                                     spectrum_kind(cfg.spectrum_power), cfg.affine());
        FA_CUDA_TRY(fa::launch(kernel, ggrid, generic_warps * 32, smem_bytes, stream, P, G));
        return FA_OK;
    }
    const int grid = std::min(total_tiles, num_sms * kCtasPerSm);
    const dim3 blk(kWarpsPerCta * 32);
    FA_CUDA_TRY(fa::launch(mel512_variant(precision, layout), grid, blk, smem_bytes, stream, P));
    return FA_OK;
}

// Shape rules shared by every entry point.  Returns false for the reference's "empty" guard
// (AudioMelSpectrogram.swift:135-137, :199-201, :349-351).
static bool shape_of(const MelPlan &p, long long n, int mode, long long expected, long long &T, long long &Tp) {
    T = p.frame_count(n, mode, mode == FA_MEL_PAD_CENTER || mode == FA_MEL_PAD_PREPADDED ? expected : -1);
    if (T <= 0 || n <= 0) return false;
    Tp = mode == FA_MEL_LEGACY_COMPUTE ? T : ceil_to(T, p.cfg.pad_to);
    return true;
}

int clip_shape(const MelPlan &p, long long n, int mode, long long expected, long long out_len, long long &T,
               long long &Tp, long long *mel_length, long long *num_frames) {
    if (!shape_of(p, n, mode, expected, T, Tp)) {
        T = 0;
        Tp = mode == FA_MEL_LEGACY_COMPUTE ? 0 : 1;
    }
    if (mel_length) *mel_length = T;
    if (num_frames) *num_frames = Tp;
    if (out_len < Tp * p.cfg.n_mels) {
        fa::set_error("mel output needs %lld floats, buffer has %lld", Tp * p.cfg.n_mels, out_len);
        return FA_OUTPUT_TOO_SMALL;
    }
    return FA_OK;
}

int MelPlan::compute_device(const float *d_in, long long n, float last, int mode, long long expected, int layout,
                            float *d_out_buf, long long out_len, long long *mel_length, long long *num_frames,
                            cudaStream_t stream) {
    long long T, Tp;
    int st = clip_shape(*this, n, mode, expected, out_len, T, Tp, mel_length, num_frames);
    if (st != FA_OK) return st;
    if (T == 0) {
        if (Tp) FA_CUDA_TRY(cudaMemsetAsync(d_out_buf, 0, cfg.n_mels * sizeof(float), stream));
        return FA_OK;
    }
    st = units.reserve(unit_bytes(1));
    if (st != FA_OK) return st;
    if (Tp > T) FA_CUDA_TRY(cudaMemsetAsync(d_out_buf, 0, Tp * cfg.n_mels * sizeof(float), stream));
    units.host.data()[0] = MelUnit{0, n, 0, Tp, 0, T, last, 0};
    st = units.upload(sizeof(MelUnit), stream);
    if (st != FA_OK) return st;
    return launch(units.device.data(), units.host.data(), 1, false, d_in, d_out_buf, mode, layout, stream);
}

int MelPlan::launch_clip(const float *d_in, long long n, long long T, int layout, float *d_out_buf, cudaStream_t stream) {
    if (T <= 0) return FA_OK;
    int st = units.reserve(unit_bytes(1));
    if (st != FA_OK) return st;
    units.host.data()[0] = MelUnit{0, n, 0, T, 0, T, 0.0f, 0};
    st = units.upload(sizeof(MelUnit), stream);
    if (st != FA_OK) return st;
    return launch(units.device.data(), units.host.data(), 1, false, d_in, d_out_buf, FA_MEL_PAD_CENTER, layout, stream);
}

int MelPlan::compute_batch_device(const float *d_in, const int64_t *offsets, int count, const float *last, int mode,
                                  int layout, float *d_out_buf, const int64_t *out_offsets, int64_t *mel_lengths,
                                  int64_t *num_frames, cudaStream_t stream) {
    int st = units.reserve(unit_bytes(count));
    if (st != FA_OK) return st;
    MelUnit *h_units = units.host.data();
    int used = 0;
    for (int i = 0; i < count; ++i) {
        const long long n = offsets[i + 1] - offsets[i];
        long long T, Tp;
        clip_shape(*this, n, mode, -1, kUnchecked, T, Tp, nullptr, nullptr);
        if (mel_lengths) mel_lengths[i] = T;
        if (num_frames) num_frames[i] = Tp;
        if (T == 0) {
            if (Tp) FA_CUDA_TRY(cudaMemsetAsync(d_out_buf + out_offsets[i], 0, cfg.n_mels * sizeof(float), stream));
            continue;
        }
        if (Tp > T) FA_CUDA_TRY(cudaMemsetAsync(d_out_buf + out_offsets[i], 0, Tp * cfg.n_mels * sizeof(float), stream));
        h_units[used++] = MelUnit{offsets[i], n, out_offsets[i], Tp, 0, T, last ? last[i] : 0.0f, 0};
    }
    if (!used) return FA_OK;
    number_tiles(h_units, used);
    st = units.upload(used * sizeof(MelUnit), stream);
    if (st != FA_OK) return st;
    return launch(units.device.data(), h_units, used, false, d_in, d_out_buf, mode, layout, stream);
}

} // namespace mel
} // namespace fa
