// Per-lane math of the fused log-mel kernel (nFFT = 512), written so that the SAME source compiles for the
// device (mel_kernels.cu) and for the host lane-emulator used by the CPU test-suite (tests/emul/mel_emul.cpp):
// every function takes the lane id explicitly, touches "shared memory" only through the pointers it is given,
// and keeps no state between phases other than the read-only LaneTables.
//
// Reference being re-implemented: Sources/FluidAudio/Shared/AudioMelSpectrogram.swift:404-453 (frame loop),
// :459-481 (512-point DFT of a real frame, power of bins 0..256), :432-452 (filterbank mat-vec + log).
//
// Algorithm (one warp per frame):
//   real frame x[0..512) (float32: window * pre-emphasised sample, exactly the reference's vDSP_vmul)
//   z[m] = x[2m] + i x[2m+1], m < 256                                     (even/odd packing)
//   Z = FFT256(z): radix 8 x 8 x 4 decimation in frequency in FP64, through shared memory, __syncwarp between passes
//   X[b] = E[b] + W512^b O[b],  E = (Z[b] + conj Z[256-b]) / 2,  O = (Z[b] - conj Z[256-b]) / (2i)      (FP64)
//   power[b] = fl32(Re X)^2 + fl32(Im X)^2 in float32, b = 0..256
//   The last radix-4 pass and the recombination are ONE register-resident step: a lane computes the two radix-4
//   butterflies whose outputs are each other's mirror images (k and 256-k), so Z never goes back to shared memory.
//
// Why FP64 for the transform: the reference's DFT (vDSP_DFT_zop) is float32, and ANY float32 FFT carries rounding
// noise of ~0.5 ulp of the frame's largest spectral line in every bin.  On input with 60 dB of dynamic range that
// alone moves weak log-mel bins by up to ~1e-4, so two correct float32 implementations cannot be compared to
// 1e-4.  Evaluating the transform in FP64 and rounding once reproduces the implementation-independent value (the
// oracle's definition) to ~1e-6 in the log domain.  The kernel is instruction-issue bound, the FP64 pipe is not the
// limiter (profiles/), so this costs little.
//
// TWO value types run through the SAME code (template parameter V):
//   V = double  one frame per warp, transform in FP64 (the parity default, see above);
//   V = f32x2   TWO frames per warp, each value a pair (frame A, frame B) of float32 in one 64-bit register pair,
//               every butterfly a pair of independent float32 operations (fa_common.cuh: FADD / FMUL / FFMA per frame on
//               sm_90), twiddles exact-rounded per-lane scalars
//               held in registers.  Same element size (16 bytes), same layouts, same index math as the FP64 path;
//               FP32 instead of FP64 arithmetic per frame.  This is what the reference's own float32 vDSP_DFT does numerically
//               (float32 noise floor: up to ~1e-4 on weak log-mel bins against the exactly rounded transform).
//
// Shared-memory layouts of the 256 complex values (16-byte elements; a warp-wide 16-byte access is 4 wavefronts
// when every 8 consecutive lanes hit 8 distinct 16-byte banks):
//   A  (pass 1 out / pass 2 in):  element idx            at idx + 4*(idx>>5)          = l + 36 q
//   B  (pass 2 out / pass 3 in):  z_{q,q2}[h]            at 74 h + 9 q + q2
// Twiddles are produced by recurrence in FP64 from one per-lane root per pass (W256^l, W32^(l&3), W512^l).  The
// kernel is bound by shared-memory wavefronts (profiles/r01c_mel.md: the three transposes of 256 complex doubles cost
// ~200 of ~330 wavefronts per frame), the FP64 pipe has headroom: twiddle tables in shared memory were measured and
// bought nothing (80 fewer FP64 instructions, 67 more wavefronts per frame).
// The recombination handles the bin pair (b, 256-b) together — both need only Z[b] and Z[256-b]:
//   2 X[b] = S + T,  2 X[256-b] = conj(S - T),  S = Z[b] + conj Z[256-b],  T = W512^b * (D.y, -D.x),  D = Z[b] - conj Z[256-b]
// — works on 2X (no multiplications by 1/2) and stores 4*|X|^2; the plan hands the kernel the filterbank weights
// times 1/4, which gives bit-identical products (power-of-two scalings commute with rounding).
#pragma once

#include "fa_common.cuh"
#include <math.h>
#include <stdint.h>

namespace fa {
namespace mel {

constexpr int kNfft = 512;
constexpr int kHalf = 256;
constexpr int kBins = 257;
constexpr int kFftPad = 304;      // complex values per warp buffer (max layout extent 296 + Z[0] mirror at 288)
constexpr int kTileFrames = 16;   // frames per CTA tile; the mel stage maps 32 / kTileFrames mel bins onto one warp
constexpr int kWarpsPerCta = 8;   // warps of a mel512_kernel CTA, for which the plan deals out the filterbank schedule
// Power tile: one row per frame PAIR, the two frames' values of a bin side by side: row[2 * bin + slot], slot = frame & 1.
// The float32-pair transform stores both frames of a bin with ONE 64-bit store, and the filterbank stage runs two frames
// per lane, both multiplied by the same weight.  Row stride 524 floats = 2 x 260 bins + 4: 16-byte
// aligned and = 12 (mod 32) banks, so the 8 lanes (pairs) of a quarter-warp reading the same bin quad hit disjoint banks.
constexpr int kPairStride = 524;
// Inside a pair row bin b sits at position pow_pos(b) = b ^ ((b >> 4) & 3): the two low bits are XORed with bits 4-5, a
// permutation INSIDE each aligned bin quad (the filterbank stage still reads whole quads at 4 * Q; the plan permutes the
// packed weights the same way).  Pass 3 stores bins k0 + 64 k2 with k0 = a + 8 j over the lanes of a quarter-warp: without
// the swizzle they hit only two 8-byte bank pairs (4-way conflicts, 24 excess wavefronts per frame on the pipe that bounds
// the kernel); with it the eight lanes hit eight distinct ones.  For a lane the XOR mask is a constant, so the swizzled
// store positions are k0s + 64 k2 and kc0s - 64 k2 with two per-lane integers.
FA_HD int pow_pos(int bin) { return bin ^ ((bin >> 4) & 3); }

struct alignas(8) cpx {
    float x, y;
};

// ---------------------------------------------------------------------------------------------- value types
// f32x2: the float32 values of two frames (a = even frame, b = odd frame of the warp's pair) in one register pair.
struct alignas(8) f32x2 {
    float a, b;
};

#if defined(__CUDA_ARCH__)
__device__ __forceinline__ float2 as_f2(f32x2 v) { return make_float2(v.a, v.b); }
__device__ __forceinline__ f32x2 as_v(float2 v) {
    f32x2 r;
    r.a = v.x;
    r.b = v.y;
    return r;
}
#endif

// generic arithmetic: vadd / vsub / vneg, vmul_s (value x per-lane scalar), vfma_s (a * s + c), vfnma_s (c - a * s)
FA_HD double vadd(double x, double y) { return x + y; }
FA_HD double vsub(double x, double y) { return x - y; }
FA_HD double vneg(double x) { return -x; }
FA_HD double vmul_s(double x, double s) { return x * s; }
FA_HD double vfma_s(double a, double s, double c) { return a * s + c; }
FA_HD double vfnma_s(double a, double s, double c) { return c - a * s; }

FA_HD f32x2 vneg(f32x2 x) {
    f32x2 r;
    r.a = -x.a;
    r.b = -x.b;
    return r;
}
#if defined(__CUDA_ARCH__)
// each one FADD / FMUL / FFMA per frame, rounded exactly as the host emulator's scalar expressions below
__device__ __forceinline__ f32x2 vadd(f32x2 x, f32x2 y) { return as_v(fadd2_rn(as_f2(x), as_f2(y))); }
__device__ __forceinline__ f32x2 vsub(f32x2 x, f32x2 y) { return as_v(fadd2_rn(as_f2(x), as_f2(vneg(y)))); }
__device__ __forceinline__ f32x2 vmul_s(f32x2 x, float s) { return as_v(fmul2_rn(as_f2(x), make_float2(s, s))); }
__device__ __forceinline__ f32x2 vfma_s(f32x2 a, float s, f32x2 c) {
    return as_v(ffma2_rn(as_f2(a), make_float2(s, s), as_f2(c)));
}
__device__ __forceinline__ f32x2 vfnma_s(f32x2 a, float s, f32x2 c) {
    return as_v(ffma2_rn(as_f2(vneg(a)), make_float2(s, s), as_f2(c)));
}
#else
inline f32x2 vadd(f32x2 x, f32x2 y) { return f32x2{x.a + y.a, x.b + y.b}; }
inline f32x2 vsub(f32x2 x, f32x2 y) { return f32x2{x.a - y.a, x.b - y.b}; }
inline f32x2 vmul_s(f32x2 x, float s) { return f32x2{x.a * s, x.b * s}; }
inline f32x2 vfma_s(f32x2 a, float s, f32x2 c) { return f32x2{fmaf(a.a, s, c.a), fmaf(a.b, s, c.b)}; }
inline f32x2 vfnma_s(f32x2 a, float s, f32x2 c) { return f32x2{fmaf(-a.a, s, c.a), fmaf(-a.b, s, c.b)}; }
#endif

template <typename V>
struct vtraits;
template <>
struct vtraits<double> {
    typedef double scalar;        // twiddle component type
    static constexpr int kFrames = 1;
};
template <>
struct vtraits<f32x2> {
    typedef float scalar;
    static constexpr int kFrames = 2;
};

// one complex value of the transform as it sits in shared memory: 16 bytes for both value types
template <typename V>
struct alignas(16) cpxv {
    V x, y;
};
typedef cpxv<double> cpxd;
struct cpxs {   // per-lane scalar twiddle of the float32 path
    float x, y;
};

// Constants a lane needs for every frame it processes; loaded once per kernel.
struct LaneCommon {
    float win[16];     // window coefficient at buffer positions j = 2(l+32r) [slot 2r] and j+1 [slot 2r+1]
    uint32_t in_win;   // bit s set  <=>  slot s lies inside [off, off+win)
    int a1, a2, k0;    // layout-B addresses of the lane's two mirror-image radix-4 butterflies; first output index
    int k0s, kc0s;     // swizzled power-row positions: bin k0 + 64 k2 -> k0s + 64 k2, bin 256 - k0 - 64 k2 -> kc0s - 64 k2
};
template <typename V>
struct LaneTables;
template <>
struct LaneTables<double> : LaneCommon {
    cpxd w256;         // W256^l        (pass 1 root; powers by FP64 recurrence)
    cpxd w32;          // W32^(l & 3)   (pass 2 root)
    cpxd wk0;          // W512^k0       (recombination root of this lane's first butterfly)
};
template <>
struct LaneTables<f32x2> : LaneCommon {
    cpxs tw1[8];       // W256^(l q), q = 1..7, exactly rounded from FP64 ([0] unused)
    cpxs tw2[8];       // W32^((l & 3) q2), q2 = 1..7
    cpxs wk[4];        // W512^(k0 + 64 k2), k2 = 0..3
};

// Pass 3 + recombination: which two of the 64 radix-4 butterflies a lane owns.  Butterfly c = 8a + b reads
// z_{c}[h] (layout B) and produces Z[k0 + 64 k2], k0 = a + 8b.  The mirror bins 256 - k come out of the butterfly
// with k0' = 64 - k0: c' = 8(8-a) + (7-b) for a >= 1, c' = (8-b) mod 8 for a = 0.  Lanes 8..31 own (l, mirror(l)),
// lanes 1..3 own (1,7) (2,6) (3,5), lanes 4..7 own (32,39) .. (35,36), lane 0 owns the two self-mirrored butterflies
// 0 and 4.  Both 16-byte loads of a quarter-warp hit eight distinct banks ((a + b + 2h) mod 8).
FA_HD void lane_butterflies(int l, int &c1, int &c2) {
    if (l >= 8) {
        c1 = l;
        c2 = 8 * (8 - (l >> 3)) + (7 - (l & 7));
    } else if (l >= 4) {
        c1 = 32 + (l - 4);
        c2 = 39 - (l - 4);
    } else if (l >= 1) {
        c1 = l;
        c2 = 8 - l;
    } else {
        c1 = 0;
        c2 = 4;
    }
}

FA_HD cpxd unit_root(int k, int n) {   // exp(-2 pi i k / n) in FP64
    const double a = -6.283185307179586476925286766559 * (double)k / (double)n;
    cpxd r;
    r.x = cos(a);
    r.y = sin(a);
    return r;
}
FA_HD cpxs unit_root_f(int k, int n) {   // the same, rounded once to float32
    const cpxd d = unit_root(k, n);
    cpxs r;
    r.x = (float)d.x;
    r.y = (float)d.y;
    return r;
}

// win_tab[512]: window value per buffer position (0 outside the window), in_tab[512]: 1 inside the window.
FA_HD void load_lane_common(int l, const float *win_tab, const uint8_t *in_tab, LaneCommon &T) {
    T.in_win = 0;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int j = 2 * (l + 32 * r);
        T.win[2 * r] = win_tab[j];
        T.win[2 * r + 1] = win_tab[j + 1];
        if (in_tab[j]) T.in_win |= 1u << (2 * r);
        if (in_tab[j + 1]) T.in_win |= 1u << (2 * r + 1);
    }
    int c1, c2;
    lane_butterflies(l, c1, c2);
    T.a1 = 9 * (c1 >> 3) + (c1 & 7);
    T.a2 = 9 * (c2 >> 3) + (c2 & 7);
    T.k0 = (c1 >> 3) + 8 * (c1 & 7);
    T.k0s = pow_pos(T.k0);
    T.kc0s = pow_pos(kHalf - T.k0);
}
FA_HD void load_lane_tables(int l, const float *win_tab, const uint8_t *in_tab, LaneTables<double> &T) {
    load_lane_common(l, win_tab, in_tab, T);
    T.w256 = unit_root(l, 256);
    T.w32 = unit_root(l & 3, 32);
    T.wk0 = unit_root(T.k0, 512);
}
FA_HD void load_lane_tables(int l, const float *win_tab, const uint8_t *in_tab, LaneTables<f32x2> &T) {
    load_lane_common(l, win_tab, in_tab, T);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        T.tw1[q] = unit_root_f((l * q) & 255, 256);
        T.tw2[q] = unit_root_f(((l & 3) * q) & 31, 32);
    }
#pragma unroll
    for (int k2 = 0; k2 < 4; ++k2) T.wk[k2] = unit_root_f(T.k0 + 64 * k2, 512);
}

FA_HD cpxd cmul(cpxd a, cpxd b) {
    cpxd r;
    r.x = a.x * b.x - a.y * b.y;
    r.y = a.x * b.y + a.y * b.x;
    return r;
}

// forward 4-point DFT, in place, natural order
template <typename V>
FA_HD void dft4(V &r0, V &i0, V &r1, V &i1, V &r2, V &i2, V &r3, V &i3) {
    const V ar = vadd(r0, r2), ai = vadd(i0, i2);
    const V br = vsub(r0, r2), bi = vsub(i0, i2);
    const V cr = vadd(r1, r3), ci = vadd(i1, i3);
    const V dr = vsub(r1, r3), di = vsub(i1, i3);
    r0 = vadd(ar, cr);
    i0 = vadd(ai, ci);
    r2 = vsub(ar, cr);
    i2 = vsub(ai, ci);
    r1 = vadd(br, di);   // d1 + (-i)(c1 - c3)
    i1 = vsub(bi, dr);
    r3 = vsub(br, di);
    i3 = vadd(bi, dr);
}

// forward 8-point DFT, in place, natural order (decimation in frequency: 4 radix-2 + two 4-point DFTs)
template <typename V>
FA_HD void dft8(V (&re)[8], V (&im)[8]) {
    typedef typename vtraits<V>::scalar S;
    const S kS = (S)0.70710678118654752440;
    V er0 = vadd(re[0], re[4]), ei0 = vadd(im[0], im[4]);
    V er1 = vadd(re[1], re[5]), ei1 = vadd(im[1], im[5]);
    V er2 = vadd(re[2], re[6]), ei2 = vadd(im[2], im[6]);
    V er3 = vadd(re[3], re[7]), ei3 = vadd(im[3], im[7]);
    V or0 = vsub(re[0], re[4]), oi0 = vsub(im[0], im[4]);
    const V xr1 = vsub(re[1], re[5]), xi1 = vsub(im[1], im[5]);
    const V xr2 = vsub(re[2], re[6]), xi2 = vsub(im[2], im[6]);
    const V xr3 = vsub(re[3], re[7]), xi3 = vsub(im[3], im[7]);
    V or1 = vmul_s(vadd(xr1, xi1), kS), oi1 = vmul_s(vsub(xi1, xr1), kS);          // * (1 - i)/sqrt2
    V or2 = xi2, oi2 = vneg(xr2);                                                  // * (-i)
    V or3 = vmul_s(vsub(xi3, xr3), kS), oi3 = vmul_s(vadd(xr3, xi3), (S)(-kS));    // * (-1 - i)/sqrt2
    dft4(er0, ei0, er1, ei1, er2, ei2, er3, ei3);
    dft4(or0, oi0, or1, oi1, or2, oi2, or3, oi3);
    re[0] = er0; im[0] = ei0;
    re[2] = er1; im[2] = ei1;
    re[4] = er2; im[4] = ei2;
    re[6] = er3; im[6] = ei3;
    re[1] = or0; im[1] = oi0;
    re[3] = or1; im[3] = oi1;
    re[5] = or2; im[5] = oi2;
    re[7] = or3; im[7] = oi3;
}

// multiply element q by root^q, q = 1..7, and hand the product to `emit(q, value)`.
// FP64: the powers are built as a depth-3 tree (w2 = w*w, w3 = w2*w, w4 = w2*w2, w5 = w4*w, w6 = w4*w2, w7 = w4*w3) to
// keep the dependent chain short.  float32 pairs: the seven twiddles are exact-rounded scalars in registers.
template <typename Emit>
FA_HD void twiddle_emit(double (&re)[8], double (&im)[8], cpxd root, Emit emit) {
    cpxd p[8];
    p[1] = root;
    p[2] = cmul(root, root);
    p[3] = cmul(p[2], root);
    p[4] = cmul(p[2], p[2]);
    p[5] = cmul(p[4], root);
    p[6] = cmul(p[4], p[2]);
    p[7] = cmul(p[4], p[3]);
    cpxd v;
    v.x = re[0];
    v.y = im[0];
    emit(0, v);
#pragma unroll
    for (int q = 1; q < 8; ++q) {
        v.x = re[q] * p[q].x - im[q] * p[q].y;
        v.y = re[q] * p[q].y + im[q] * p[q].x;
        emit(q, v);
    }
}
template <typename Emit>
FA_HD void twiddle_emit(f32x2 (&re)[8], f32x2 (&im)[8], const cpxs (&tw)[8], Emit emit) {
    cpxv<f32x2> v;
    v.x = re[0];
    v.y = im[0];
    emit(0, v);
#pragma unroll
    for (int q = 1; q < 8; ++q) {
        v.x = vfnma_s(im[q], tw[q].y, vmul_s(re[q], tw[q].x));
        v.y = vfma_s(im[q], tw[q].x, vmul_s(re[q], tw[q].y));
        emit(q, v);
    }
}
FA_HD void twiddle_pass1(int l, double (&re)[8], double (&im)[8], const LaneTables<double> &T, cpxd *buf) {
    twiddle_emit(re, im, T.w256, [&](int q, cpxd v) { buf[l + 36 * q] = v; });
}
FA_HD void twiddle_pass1(int l, f32x2 (&re)[8], f32x2 (&im)[8], const LaneTables<f32x2> &T, cpxv<f32x2> *buf) {
    twiddle_emit(re, im, T.tw1, [&](int q, cpxv<f32x2> v) { buf[l + 36 * q] = v; });
}
FA_HD void twiddle_pass2(int base, double (&re)[8], double (&im)[8], const LaneTables<double> &T, cpxd *buf) {
    twiddle_emit(re, im, T.w32, [&](int q2, cpxd v) { buf[base + q2] = v; });
}
FA_HD void twiddle_pass2(int base, f32x2 (&re)[8], f32x2 (&im)[8], const LaneTables<f32x2> &T, cpxv<f32x2> *buf) {
    twiddle_emit(re, im, T.tw2, [&](int q2, cpxv<f32x2> v) { buf[base + q2] = v; });
}

// windowed samples of the lane's slot r -> transform values.  pf -> frame (A), pf + hop -> frame B of the pair.
FA_HD void widen(float a, float b, float, float, double &re, double &im) {
    re = (double)a;
    im = (double)b;
}
FA_HD void widen(float a, float b, float a2, float b2, f32x2 &re, f32x2 &im) {
    re.a = a;
    re.b = a2;
    im.a = b;
    im.b = b2;
}

// Pass 1.  pf -> pre-emphasised sample at buffer position j = 0 of this frame (8-byte aligned, hop even).
// Window product in float32 (the reference's vDSP_vmul), then widened (FP64) or paired with the next frame's (f32x2).
// Output layout A.
// kMidFull: the window covers buffer positions [64, 448), so slots r = 1..6 of every lane are inside it and only the
// first and last slot need the in-window select (win 400 centred: positions 56..455).
template <bool kMidFull, typename V>
FA_HD void pass1(int l, const float *pf, int hop, const LaneTables<V> &T, cpxv<V> *buf) {
    V re[8], im[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const int j = 2 * (l + 32 * r);
#if defined(__CUDA_ARCH__)
        const float2 v = *reinterpret_cast<const float2 *>(pf + j);   // one 64-bit shared load (LDS.64)
        float2 u = v;
        if (vtraits<V>::kFrames == 2) u = *reinterpret_cast<const float2 *>(pf + hop + j);
#else
        const cpx v = *reinterpret_cast<const cpx *>(pf + j);
        cpx u = v;
        if (vtraits<V>::kFrames == 2) u = *reinterpret_cast<const cpx *>(pf + hop + j);
#endif
        float a = T.win[2 * r] * v.x, b = T.win[2 * r + 1] * v.y;
        float a2 = T.win[2 * r] * u.x, b2 = T.win[2 * r + 1] * u.y;
        if (!kMidFull || r == 0 || r == 7) {   // outside the window the reference's buffer holds 0, whatever the sample
            const bool ia = (T.in_win >> (2 * r)) & 1u, ib = (T.in_win >> (2 * r + 1)) & 1u;
            a = ia ? a : 0.0f;
            b = ib ? b : 0.0f;
            a2 = ia ? a2 : 0.0f;
            b2 = ib ? b2 : 0.0f;
        }
        widen(a, b, a2, b2, re[r], im[r]);
    }
    dft8(re, im);
    twiddle_pass1(l, re, im, T, buf);
}

// Pass 2 is split: its output layout (B) differs from its input layout (A), every lane must finish loading first.
template <typename V>
FA_HD void pass2_load(int l, const cpxv<V> *buf, V (&re)[8], V (&im)[8]) {
    const int base = 36 * (l >> 2) + (l & 3);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        const cpxv<V> v = buf[base + 4 * r];
        re[r] = v.x;
        im[r] = v.y;
    }
}
template <typename V>
FA_HD void pass2_store(int l, const LaneTables<V> &T, V (&re)[8], V (&im)[8], cpxv<V> *buf) {
    dft8(re, im);
    const int base = 74 * (l & 3) + 9 * (l >> 2);
    twiddle_pass2(base, re, im, T, buf);
}

// Real-FFT recombination + power, one bin PAIR (b, 256 - b) per step (see the header).  prow -> this frame's slot in its
// pair row of the power tile (FP64 path: row + (frame & 1); float32 pairs: the row itself); receives 4 |X[b]|^2, b = 0..256.
FA_HD void pair_power(double zbx, double zby, double zcx, double zcy, double wx, double wy, float *prow, int ib, int ic) {
    const double sr = zbx + zcx, si = zby - zcy;             // S
    const double dr = zby + zcy, di = zcx - zbx;             // (D.y, -D.x)
    const double tr = wx * dr - wy * di, ti = wx * di + wy * dr;
    const float xr = (float)(sr + tr), xi = (float)(si + ti);    // single rounding of the exact-arithmetic DFT (x2)
    const float yr = (float)(sr - tr), yi = (float)(si - ti);
#if defined(__CUDA_ARCH__)
    prow[2 * ib] = __fadd_rn(__fmul_rn(xr, xr), __fmul_rn(xi, xi));
    prow[2 * ic] = __fadd_rn(__fmul_rn(yr, yr), __fmul_rn(yi, yi));
#else
    const float a = xr * xr, b = xi * xi, c = yr * yr, d = yi * yi;
    prow[2 * ib] = a + b;
    prow[2 * ic] = c + d;
#endif
}
FA_HD void pair_power(f32x2 zbx, f32x2 zby, f32x2 zcx, f32x2 zcy, float wx, float wy, float *prow, int ib, int ic) {
    const f32x2 sr = vadd(zbx, zcx), si = vsub(zby, zcy);
    const f32x2 dr = vadd(zby, zcy), di = vsub(zcx, zbx);
    const f32x2 tr = vfnma_s(di, wy, vmul_s(dr, wx)), ti = vfma_s(dr, wy, vmul_s(di, wx));
    const f32x2 xr = vadd(sr, tr), xi = vadd(si, ti);
    const f32x2 yr = vsub(sr, tr), yi = vsub(si, ti);
#if defined(__CUDA_ARCH__)
    const float2 pb = ffma2_rn(as_f2(xr), as_f2(xr), fmul2_rn(as_f2(xi), as_f2(xi)));
    const float2 pc = ffma2_rn(as_f2(yr), as_f2(yr), fmul2_rn(as_f2(yi), as_f2(yi)));
    *reinterpret_cast<float2 *>(prow + 2 * ib) = pb;   // (frame A, frame B) of bin ib: one 64-bit store
    *reinterpret_cast<float2 *>(prow + 2 * ic) = pc;
#else
    prow[2 * ib] = fmaf(xr.a, xr.a, xi.a * xi.a);
    prow[2 * ic] = fmaf(yr.a, yr.a, yi.a * yi.a);
    prow[2 * ib + 1] = fmaf(xr.b, xr.b, xi.b * xi.b);
    prow[2 * ic + 1] = fmaf(yr.b, yr.b, yi.b * yi.b);
#endif
}

// the four recombination roots W512^(k0 + 64 k2) of a lane
FA_HD void recombination_roots(const LaneTables<double> &T, double (&wx)[4], double (&wy)[4]) {
    const double hh = 0.70710678118654752440;
    wx[0] = T.wk0.x;
    wy[0] = T.wk0.y;
    wx[1] = hh * (wx[0] + wy[0]);   // * W8   = (1 - i)/sqrt2
    wy[1] = hh * (wy[0] - wx[0]);
    wx[2] = wy[0];                  // * W8^2 = -i
    wy[2] = -wx[0];
    wx[3] = wy[1];                  // * W8^3 = W8 * (-i)
    wy[3] = -wx[1];
}
FA_HD void recombination_roots(const LaneTables<f32x2> &T, float (&wx)[4], float (&wy)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        wx[k] = T.wk[k].x;
        wy[k] = T.wk[k].y;
    }
}

// Pass 3 fused with the recombination (see lane_butterflies): A = butterfly c1 -> Z[k0 + 64 k2], B = butterfly c2 ->
// Z[(64 - k0) + 64 k2], so bin b = k0 + 64 k2 pairs A[k2] with B[3 - k2] and W512^b = W512^k0 * W8^k2.
// Lane 0 (k0 = 0; A = Z[0], Z[64], Z[128], Z[192]; B = Z[32], Z[96], Z[160], Z[224]) pairs inside its butterflies:
// (0,256 = Z[0]) (64,192) (128,128) in slots 0..2, (32,224) in slot 3 and (96,160) in one extra step.
template <typename V>
FA_HD void pass3_post(int l, const cpxv<V> *buf, const LaneTables<V> &T, float *prow) {
    typedef typename vtraits<V>::scalar S;
    V ar[4], ai[4], br[4], bi[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) {
        const cpxv<V> u = buf[T.a1 + 74 * h], v = buf[T.a2 + 74 * h];
        ar[h] = u.x;
        ai[h] = u.y;
        br[h] = v.x;
        bi[h] = v.y;
    }
    dft4(ar[0], ai[0], ar[1], ai[1], ar[2], ai[2], ar[3], ai[3]);
    dft4(br[0], bi[0], br[1], bi[1], br[2], bi[2], br[3], bi[3]);
    const bool z = l == 0;
    const S c1 = (S)0.92387953251128675613, s1 = (S)0.38268343236508977173;
    S wx[4], wy[4];
    recombination_roots(T, wx, wy);
    // slot 0
    // (positions: see pow_pos; 64 k2 never reaches the two swizzled bits, and their mask (bits 4-5) is the lane's constant)
    pair_power(ar[0], ai[0], z ? ar[0] : br[3], z ? ai[0] : bi[3], wx[0], wy[0], prow, T.k0s, T.kc0s);
    // slot 1
    pair_power(ar[1], ai[1], z ? ar[3] : br[2], z ? ai[3] : bi[2], wx[1], wy[1], prow, T.k0s + 64, T.kc0s - 64);
    // slot 2
    pair_power(ar[2], ai[2], z ? ar[2] : br[1], z ? ai[2] : bi[1], wx[2], wy[2], prow, T.k0s + 128, T.kc0s - 128);
    // slot 3 (lane 0: bins 32 / 224, W512^32 = W16)
    const int b3 = z ? pow_pos(32) : T.k0s + 192, c3 = z ? pow_pos(224) : T.kc0s - 192;
    pair_power(z ? br[0] : ar[3], z ? bi[0] : ai[3], z ? br[3] : br[0], z ? bi[3] : bi[0], z ? c1 : wx[3],
               z ? (S)(-s1) : wy[3], prow, b3, c3);
    if (z) {                     // bins 96 / 160, W512^96 = W16^3
        pair_power(br[1], bi[1], br[2], bi[2], s1, (S)(-c1), prow, pow_pos(96), pow_pos(160));
    }
}

// Filterbank dot product over the filter's non-zero band.  Host (emulator / oracle order): float32 accumulate in bin
// order with separate multiply and add roundings.  Device: the plan aligns the band to bin quads (explicit zero
// weights), rows of the power tile are 16-byte aligned, so one step is two 16-byte shared loads and four FMAs;
// fusing the multiply-add moves the result by <= 1 ulp of the sum (the parity bar on log-mel is 1e-4).
FA_HD float mel_dot(const float *prow, const float *w, int lo, int hi) {
    float acc = 0.0f;
    const float *p = prow + lo;
    const int n = hi - lo;
    for (int b = 0; b < n; ++b) {
        const float t = w[b] * p[b];
        acc = acc + t;
    }
    return acc;
}
#if defined(__CUDACC__)
// Two frames at once out of a pair row: p4 -> (bin, slot) interleaved values of the band's first quad (two float4 per bin
// quad), w4 -> packed weights; four FFMA pairs per quad, the weight shared by both frames.
__device__ __forceinline__ float2 mel_dot_pairs(const float4 *p4, const float4 *w4, int nq) {
    float2 acc = make_float2(0.0f, 0.0f);
#pragma unroll 1
    for (int b = 0; b < nq; ++b) {
        const float4 x01 = p4[2 * b], x23 = p4[2 * b + 1], c = w4[b];
        acc = ffma2_rn(make_float2(x01.x, x01.y), make_float2(c.x, c.x), acc);
        acc = ffma2_rn(make_float2(x01.z, x01.w), make_float2(c.y, c.y), acc);
        acc = ffma2_rn(make_float2(x23.x, x23.y), make_float2(c.z, c.z), acc);
        acc = ffma2_rn(make_float2(x23.z, x23.w), make_float2(c.w, c.w), acc);
    }
    return acc;
}
// p4 / w4: first quad of the band in the power row / in the packed weights; nq quads.  Not unrolled: bands are 1..6
// quads long and the unrolled remainder ladder cost ~100 instructions per dot product (profiles/r01c_mel.md).
__device__ __forceinline__ float mel_dot_quads(const float4 *p4, const float4 *w4, int nq) {
    float acc = 0.0f;
#pragma unroll 1
    for (int b = 0; b < nq; ++b) {
        const float4 x = p4[b], c = w4[b];
        acc = fmaf(c.x, x.x, acc);
        acc = fmaf(c.y, x.y, acc);
        acc = fmaf(c.z, x.z, acc);
        acc = fmaf(c.w, x.w, acc);
    }
    return acc;
}
#endif

// log of a mel value.  Device: one MUFU.LG2 and one multiply (|error| <= ~2 ulp of the result: 4e-6 at log(2^-24),
// against the 1e-4 bar); host emulator: libm.  normal_floor: the floor is a normal float, so the argument never is a
// denormal and the denormal pre-scaling of __log2f (three more instructions) can be skipped.
// Clamped: max(v, floor) as Swift's max (AudioMelSpectrogram.swift:547) and std::max evaluate it, so a NaN mel value stays
// NaN (`v > floor ? v : floor` would turn it into log(floor)); every other value gives the same bits either way.
FA_HD float log_value(float v, float floor_, int clamped, int normal_floor = 0) {
    const float x = clamped ? (floor_ >= v ? floor_ : v) : v + floor_;
#if defined(__CUDA_ARCH__)
    float l;
    if (normal_floor) asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(x));
    else l = __log2f(x);
    return l * 0.693147180559945309417f;
#else
    (void)normal_floor;
    return logf(x);
#endif
}

// Pre-emphasis y[i] = x[i] - a x[i-1].  i == 0 uses Swift scalar arithmetic (two roundings,
// AudioMelSpectrogram.swift:373); i > 0 is vDSP_vsma = fused multiply-add (:381-387).
FA_HD float preemph_first(float x0, float last, float a) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(x0, __fmul_rn(a, last));
#else
    const float t = a * last;
    return x0 - t;
#endif
}
FA_HD float preemph_rest(float x, float xprev, float a) { return fmaf(xprev, -a, x); }

// Reflect padding of a clip of n >= 1 samples (FA_MEL_EDGE_REFLECT): the sample index audio index i reads.  These are
// the reference's clamps (StyleTTS2MelExtractor.swift:226-250, LuxTtsMelExtractor.swift:57-64), not torch's rule:
// i < 0 reads x[min(-i, n-1)], i >= n reads x[max(2n-2-i, 0)], so a clip shorter than the pad repeats its end samples
// instead of failing.  [a,b,c,d] padded by 2 reads [c,b,a,b,c,d,c,b].  The any-nFFT kernel and the CPU emulation
// (tests/emul/mel_reflect_emul.cpp) share this function.
FA_HD long long reflect_index(long long i, long long n) {
    if (i < 0) return -i < n - 1 ? -i : n - 1;
    if (i >= n) return 2 * n - 2 - i > 0 ? 2 * n - 2 - i : 0;
    return i;
}

} // namespace mel
} // namespace fa
