// VBx refinement, gamma-weighted centroids and cosine assignment in FP64 on sm_90a.
//
// Re-implements
//   Sources/FluidAudio/Diarizer/Offline/Clustering/VBxClustering.swift:167-664   (runVBx)
//   Sources/FluidAudio/Diarizer/Offline/Core/OfflineDiarizerManager.swift:613-691 (computeCentroids)
//   OfflineDiarizerManager.swift:789-883                                          (centroidScores/assignEmbeddings)
//
// All reductions over frames use a FIXED two-level order (sequential inside a chunk of frames, chunks folded in
// ascending order by one CTA), so results are bit-reproducible run to run (the reference asserts its cluster
// phase is bit-identical across repeats, OfflineDiarizerTwoPhaseTests.swift:20-33).  The reference's own sums
// come from closed-source BLAS/vDSP with unknown association, so gamma/pi/ELBO parity is to 1e-9-ish, hard
// labels exact.  The whole EM loop runs without a host round trip: a device-side `done` flag turns the kernels
// of the remaining iterations into no-ops once |dELBO| < epsilon.
#include "vbx_plan.h"

#include <algorithm>
#include <cmath>
#include <vector>

namespace fa {
namespace vbx {

constexpr int kChunks = 128;      // frame chunks for the two-level reductions (fewer when there are > 1024 speakers)
constexpr int kEThreads = 128;    // threads per CTA in the E-step
constexpr int kFChunks = 16;      // frame chunks of the two-kernel EM path
constexpr int kFusedMaxS = 64;    // speakers the two-kernel EM path handles (alpha and invL tiles live in shared memory)

// Partial sums are [chunks x S x D]: keep them bounded when AHC hands over thousands of clusters (degenerate input:
// every embedding its own speaker).  The chunk count only changes the (fixed) summation order.
static int chunks_for(int S) { return S <= 1024 ? kChunks : std::max(1, (kChunks * 1024) / S); }

struct Dev {
    int T, D, S, Tp, chunks;
    const double *x;      // [T x D] features
    const double *phi_c;  // [D] clamped psi
    double *rho;          // [T x D]
    double *rhoT;         // [D x Tp]
    double *G;            // [T]
    double *gamma;        // [T x S]
    double *pi;           // [S]
    double *invL, *alpha; // [S x D]
    double *phiTerm, *logPi, *gsum; // [S]
    double *pA;           // [chunks x S x D]
    double *pG;           // [chunks x S]
    double *pLL;          // [blocks]
    double *pPi;          // [blocks x S]
    double *elbos;        // [max_it]
    double *scal;         // [0]=sumLogInv [1]=sumInv [2]=sumAlphaSq [3]=prevElbo
    int *state;           // [0]=done [1]=iterations
    int eblocks;
    double Fa, Fb, eps;
    // two-kernel path (S <= kFusedMaxS): partials over kFChunks frame chunks, E-step partials double-buffered by iteration
    double *fA, *fG;        // [eblocks x S x D], [eblocks x S]: per-frame-block gamma^T rho and column sums of gamma
    double *fLL;            // [eblocks] per-block log-likelihood
    double *fsums[2];       // [3 x S] per speaker: sum log invL, sum invL, sum alpha^2 (double-buffered by iteration)
};

// gamma0 = softmax(7 * onehot) row-wise, then renormalise (VBxClustering.swift:190-235); rho = x * sqrt(phi);
// G = -0.5 (|x|^2 + D ln 2 pi) (:239-282)
__global__ void vbx_init_kernel(Dev d, const int *__restrict__ init, double smoothing) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= d.T) return;
    const int S = d.S;
    double *g = d.gamma + (size_t)t * S;
    const int label = init ? max(0, min(init[t], S - 1)) : -1;
    for (int s = 0; s < S; ++s) g[s] = init ? (s == label ? 1.0 : 0.0) : 1.0 / (double)S;
    if (smoothing >= 0.0) {
        double mx = -1.7976931348623157e308;
        for (int s = 0; s < S; ++s) mx = fmax(mx, g[s] * smoothing);
        double sum = 0.0;
        for (int s = 0; s < S; ++s) {
            const double e = exp(g[s] * smoothing - mx);
            g[s] = e;
            sum += e;
        }
        if (sum <= 0.0 || !isfinite(sum)) {
            for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
        } else {
            const double inv = 1.0 / sum;
            for (int s = 0; s < S; ++s) g[s] *= inv;
        }
    }
    double sum = 0.0;
    for (int s = 0; s < S; ++s) sum += g[s];
    if (sum <= 0.0 || !isfinite(sum)) {
        for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
    } else {
        const double inv = 1.0 / sum;
        for (int s = 0; s < S; ++s) g[s] *= inv;
    }
    const double *x = d.x + (size_t)t * d.D;
    double ss = 0.0;
    for (int k = 0; k < d.D; ++k) {
        const double v = x[k];
        const double r = v * sqrt(d.phi_c[k]);
        d.rho[(size_t)t * d.D + k] = r;
        d.rhoT[(size_t)k * d.Tp + t] = r;
        ss += v * v;
    }
    d.G[t] = -0.5 * (ss + (double)d.D * log(2.0 * 3.14159265358979323846));
}

// per chunk of frames: pG[c][s] = sum_t gamma[t][s], pA[c][s][k] = sum_t gamma[t][s] rho[t][k]   (:304-360)
__global__ void vbx_accumulate_kernel(Dev d) {
    if (d.state[0]) return;
    const int c = blockIdx.x;
    const int per = (d.T + d.chunks - 1) / d.chunks;
    const int t0 = c * per, t1 = min(d.T, t0 + per);
    const int SD = d.S * d.D;
    for (int o = threadIdx.x; o < SD; o += blockDim.x) {
        const int s = o / d.D, k = o % d.D;
        double acc = 0.0;
        for (int t = t0; t < t1; ++t) acc += d.gamma[(size_t)t * d.S + s] * d.rho[(size_t)t * d.D + k];
        d.pA[(size_t)c * SD + o] = acc;
    }
    for (int s = threadIdx.x; s < d.S; s += blockDim.x) {
        double acc = 0.0;
        for (int t = t0; t < t1; ++t) acc += d.gamma[(size_t)t * d.S + s];
        d.pG[(size_t)c * d.S + s] = acc;
    }
}

// single CTA: fold chunks, invL, alpha, phiTerm, log pi and the three ELBO sums   (:330-436, :496-516, :623-644)
__global__ void vbx_update_kernel(Dev d) {
    if (d.state[0]) return;
    const int S = d.S, D = d.D, SD = S * D;
    const double ratio = d.Fa / d.Fb;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        double acc = 0.0;
        for (int c = 0; c < d.chunks; ++c) acc += d.pG[(size_t)c * S + s];
        d.gsum[s] = acc;
        d.logPi[s] = log(fmax(d.pi[s], 1e-8));
    }
    __syncthreads();
    for (int o = threadIdx.x; o < SD; o += blockDim.x) {
        const int s = o / D, k = o % D;
        double acc = 0.0;
        for (int c = 0; c < d.chunks; ++c) acc += d.pA[(size_t)c * SD + o];
        const double il = 1.0 / fmax(1.0 + (ratio * d.gsum[s]) * d.phi_c[k], 1e-12);
        d.invL[o] = il;
        d.alpha[o] = (acc * il) * ratio;
    }
    __syncthreads();
    __shared__ double sh[3][256];
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        double p = 0.0;
        for (int k = 0; k < D; ++k) {
            const double a = d.alpha[s * D + k], il = d.invL[s * D + k];
            p += (a * a + il) * d.phi_c[k];
        }
        d.phiTerm[s] = p;
    }
    // ELBO sums: thread-strided partials in a fixed order, then a sequential fold by thread 0
    double l = 0.0, i2 = 0.0, a2 = 0.0;
    for (int o = threadIdx.x; o < SD; o += blockDim.x) {
        const double il = d.invL[o], a = d.alpha[o];
        l += log(il);
        i2 += il;
        a2 += a * a;
    }
    sh[0][threadIdx.x] = l;
    sh[1][threadIdx.x] = i2;
    sh[2][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.x == 0) {
        double x0 = 0, x1 = 0, x2 = 0;
        for (int i = 0; i < (int)blockDim.x; ++i) {
            x0 += sh[0][i];
            x1 += sh[1][i];
            x2 += sh[2][i];
        }
        d.scal[0] = x0;
        d.scal[1] = x1;
        d.scal[2] = x2;
    }
}

// thread per frame: log-likelihood row, soft-max -> gamma, per-CTA partial LL and partial pi   (:438-602)
// kAlphaSmem: alpha [S x D], -phiTerm/2 and log pi staged in shared memory (the normal case, S x D x 8 <= 200 KB);
// otherwise read through L2 (hundreds of speakers: same arithmetic, every warp reads the same addresses).
template <bool kAlphaSmem>
__global__ void __launch_bounds__(kEThreads) vbx_estep_kernel(Dev d) {
    if (d.state[0]) return;
    extern __shared__ double sm[];
    const int S = d.S, D = d.D;
    double *red = sm;                                        // [kEThreads]
    const double *alpha = d.alpha;
    if (kAlphaSmem) {
        double *a_s = sm + kEThreads;                        // [S x D]
        double *off_s = a_s + (size_t)S * D;                 // [S]  -0.5 phiTerm
        double *lpi_s = off_s + S;                           // [S]
        for (int o = threadIdx.x; o < S * D; o += kEThreads) a_s[o] = d.alpha[o];
        for (int s = threadIdx.x; s < S; s += kEThreads) {
            off_s[s] = d.phiTerm[s] * -0.5;
            lpi_s[s] = d.logPi[s];
        }
        __syncthreads();
        alpha = a_s;
    }
    const double *off = kAlphaSmem ? sm + kEThreads + (size_t)S * D : nullptr;
    const double *lpi = kAlphaSmem ? off + S : nullptr;
    const int t = blockIdx.x * kEThreads + threadIdx.x;
    double ll = 0.0;
    if (t < d.T) {
        double *g = d.gamma + (size_t)t * S;
        const double Gt = d.G[t];
        double mx = -1.7976931348623157e308;
        for (int s = 0; s < S; ++s) {
            double acc = 0.0;
            const double *a = alpha + (size_t)s * D;
            for (int k = 0; k < D; ++k) acc += d.rhoT[(size_t)k * d.Tp + t] * a[k];
            const double o_s = kAlphaSmem ? off[s] : d.phiTerm[s] * -0.5;
            const double l_s = kAlphaSmem ? lpi[s] : d.logPi[s];
            const double v = ((acc + o_s) + Gt) * d.Fa + l_s;
            g[s] = v;
            mx = fmax(mx, v);
        }
        double sum = 0.0;
        for (int s = 0; s < S; ++s) {
            const double e = exp(g[s] - mx);
            g[s] = e;
            sum += e;
        }
        if (sum <= 0.0 || !isfinite(sum)) {
            for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
            ll = mx;
        } else {
            const double inv = 1.0 / sum;
            for (int s = 0; s < S; ++s) g[s] *= inv;
            ll = mx + log(sum);
        }
    }
    red[threadIdx.x] = ll;
    __syncthreads();
    if (threadIdx.x == 0) {
        double acc = 0.0;
        for (int i = 0; i < kEThreads; ++i) acc += red[i];
        d.pLL[blockIdx.x] = acc;
    }
    // partial pi: column sums of this CTA's rows, sequential over rows
    // (the barrier above also makes every gamma row of this CTA visible to all of its threads)
    const int t0 = blockIdx.x * kEThreads, t1 = min(d.T, t0 + kEThreads);
    for (int s = threadIdx.x; s < S; s += kEThreads) {
        double acc = 0.0;
        for (int tt = t0; tt < t1; ++tt) acc += d.gamma[(size_t)tt * S + s];
        d.pPi[(size_t)blockIdx.x * S + s] = acc;
    }
}

// single CTA: LL, pi, ELBO, convergence   (:578-661)
__global__ void vbx_finish_kernel(Dev d, int iteration) {
    if (d.state[0]) return;
    const int S = d.S;
    __shared__ double piSum;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        double acc = 0.0;
        for (int b = 0; b < d.eblocks; ++b) acc += d.pPi[(size_t)b * S + s];
        d.pi[s] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ps = 0.0;
        for (int s = 0; s < S; ++s) ps += d.pi[s];
        piSum = ps;
    }
    __syncthreads();
    const double ps = piSum;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        if (ps > 0.0 && isfinite(ps)) d.pi[s] *= (1.0 / ps);
        else d.pi[s] = 1.0 / (double)S;
    }
    if (threadIdx.x == 0) {
        double ll = 0.0;
        for (int b = 0; b < d.eblocks; ++b) ll += d.pLL[b];
        const double count = (double)(S * d.D);
        const double elbo = ll + d.Fb * 0.5 * (d.scal[0] - d.scal[1] - d.scal[2] + count);
        d.elbos[iteration] = elbo;
        d.state[1] = iteration + 1;
        if (iteration > 0 && fabs(elbo - d.scal[3]) < d.eps) d.state[0] = 1;
        d.scal[3] = elbo;
    }
}


// ---- two-kernel EM iteration (the normal case: a handful of speakers) -----------------------------------------------
// The EM loop is tiny (C3: 2 x 10 MFLOP per iteration) and was bound by LATENCY: one-accumulator chains of hundreds of
// dependent loads and a single CTA folding 128 partials.  Here every chain carries kSG = 8 speakers at once (eight
// independent FP64 accumulators per thread: one load feeds eight FMAs) and no fold is longer than the number of frame
// blocks, spread over S CTAs:
//   vbx_update_kernel2 (S CTAs)      CTA s: pi and N_s from the per-block column sums, ELBO of the previous iteration and
//                                    the convergence test (VBxClustering.swift:578-661), then A[s][.] folded over the
//                                    frame blocks, invL, alpha, phi_s, log pi_s and this speaker's share of the ELBO sums
//                                    (:304-436, :496-516, :623-644).
//   vbx_estep_kernel2 (T/128 CTAs)   thread per frame: log-likelihood row (k outer, speakers in registers), soft-max,
//                                    gamma (:438-576); then, with the block's new gamma rows in shared memory, the block's
//                                    partial sums for the NEXT update: column sums, LL, gamma^T rho (thread per dimension).
// All sums keep a FIXED order (k ascending; frames ascending inside a block; blocks ascending): bit-reproducible.
constexpr int kSG = 8;   // speakers per register group

// partial sums of one frame block from the gamma rows in shared memory: fG[b][s], fA[b][s][k]
// tile: optional shared-memory copy of the block's rho, k-major with stride kEThreads + 1 (tile[k * (kEThreads + 1) + r]);
// nullptr = read rho from global memory
__device__ __forceinline__ void vbx_block_partials(const Dev &d, const double *g_s, int t0, int rows, int b,
                                                   const double *tile = nullptr) {
    const int S = d.S, D = d.D, tid = threadIdx.x;
    for (int s = tid; s < S; s += kEThreads) {
        double acc = 0.0;
        for (int r = 0; r < rows; ++r) acc += g_s[r * S + s];
        d.fG[(size_t)b * S + s] = acc;
    }
    for (int k = tid; k < D; k += kEThreads) {
        const double *rk = d.rho + (size_t)t0 * D + k;
        for (int s0 = 0; s0 < S; s0 += kSG) {
            double acc[kSG];
#pragma unroll
            for (int q = 0; q < kSG; ++q) acc[q] = 0.0;
            for (int r = 0; r < rows; ++r) {
                const double x = tile ? tile[k * (kEThreads + 1) + r] : rk[(size_t)r * D];
                const double *g = g_s + r * S + s0;
#pragma unroll
                for (int q = 0; q < kSG; ++q)
                    if (s0 + q < S) acc[q] += g[q] * x;
            }
#pragma unroll
            for (int q = 0; q < kSG; ++q)
                if (s0 + q < S) d.fA[((size_t)b * S + s0 + q) * D + k] = acc[q];
        }
    }
}

// partials of the INITIAL gamma (before the first update)
__global__ void __launch_bounds__(kEThreads) vbx_partials0_kernel(Dev d) {
    extern __shared__ double sm[];
    const int S = d.S, b = blockIdx.x, t0 = b * kEThreads, rows = min(kEThreads, d.T - t0);
    for (int i = threadIdx.x; i < rows * S; i += kEThreads) sm[i] = d.gamma[(size_t)t0 * S + i];
    __syncthreads();
    vbx_block_partials(d, sm, t0, rows, b);
}

// closing == 1: only the pi / ELBO bookkeeping of the last E-step (after max_iterations launches)
// Convergence: the launch that finds it stores its own `it` (>= 2) in state[0], which turns every later kernel into a
// no-op.  This kernel's S CTAs test it at entry, so they skip only when an EARLIER launch converged: a CTA of the
// converging launch that starts after CTA 0's store must still write its pi.
__global__ void __launch_bounds__(kEThreads) vbx_update_kernel2(Dev d, int it, int closing) {
    const int conv = d.state[0];
    if (conv && conv < it) return;   // converged in an earlier launch
    __shared__ double pi_sh[kFusedMaxS];
    __shared__ double red[kEThreads];
    __shared__ double scal[4];
    __shared__ int done_sh;
    const int S = d.S, D = d.D, tid = threadIdx.x, s = blockIdx.x, nb = d.eblocks;
    const int prev = (it + 1) & 1, cur = it & 1;
    // column sums of gamma_it per speaker and the log-likelihood, frame blocks ascending.  The per-block partials are
    // first staged in shared memory by ALL threads (coalesced, one latency), then summed in block order from there:
    // the same fixed order as a sequential fold, without 79 dependent global loads per speaker on one thread.
    __shared__ double stage[64 * (kFusedMaxS + 1)];
    for (int c = tid; c < S; c += kEThreads) pi_sh[c] = 0.0;
    double ll = 0.0;   // thread 0 only
    if (tid == 0) done_sh = 0;
    for (int b0 = 0; b0 < nb; b0 += 64) {
        const int cnt = min(64, nb - b0);
        __syncthreads();
        for (int i = tid; i < cnt * S; i += kEThreads) stage[i] = d.fG[(size_t)b0 * S + i];
        if (it > 0)
            for (int i = tid; i < cnt; i += kEThreads) stage[64 * S + i] = d.fLL[b0 + i];
        __syncthreads();
        for (int c = tid; c < S; c += kEThreads) {
            double v = pi_sh[c];
            for (int b = 0; b < cnt; ++b) v += stage[b * S + c];
            pi_sh[c] = v;
        }
        if (tid == 0 && it > 0)
            for (int b = 0; b < cnt; ++b) ll += stage[64 * S + b];
    }
    __syncthreads();
    if (tid == 0) {
        double ps = 0.0;
        for (int c = 0; c < S; ++c) ps += pi_sh[c];
        scal[0] = ps;
        if (it > 0) {   // ELBO_{it-1} (:623-647) and the convergence test (:653-659)
            double x0 = 0.0, x1 = 0.0, x2 = 0.0;
            for (int c = 0; c < S; ++c) {
                x0 += d.fsums[prev][3 * c];
                x1 += d.fsums[prev][3 * c + 1];
                x2 += d.fsums[prev][3 * c + 2];
            }
            const double elbo = ll + d.Fb * 0.5 * (x0 - x1 - x2 + (double)(S * D));
            scal[1] = elbo;
            if (closing || (it > 1 && fabs(elbo - d.elbos[it - 2]) < d.eps)) done_sh = 1;
        }
    }
    __syncthreads();
    const double ps = scal[0];
    const double Ns = pi_sh[s];                                   // N_s = sum_t gamma_ts (:304-328)
    const bool ok = ps > 0.0 && isfinite(ps);
    const double pi_s = it == 0 ? d.pi[s] : (ok ? Ns * (1.0 / ps) : 1.0 / (double)S);   // pi (:578-621); 1/S initially (:237)
    if (it > 0 && tid == 0) {
        d.pi[s] = pi_s;
        if (s == 0) {
            d.elbos[it - 1] = scal[1];
            d.state[1] = it;
            if (done_sh && !closing) d.state[0] = it;
        }
    }
    if (done_sh || closing) return;
    // A[s][k] over the frame blocks (ascending), invL, alpha
    const double ratio = d.Fa / d.Fb;
    double p_part = 0.0, l_part = 0.0, i_part = 0.0, a_part = 0.0;
    for (int k = tid; k < D; k += kEThreads) {
        double acc = 0.0;
#pragma unroll 16
        for (int b = 0; b < nb; ++b) acc += d.fA[((size_t)b * S + s) * D + k];
        const double il = 1.0 / fmax(1.0 + (ratio * Ns) * d.phi_c[k], 1e-12);
        const double al = (acc * il) * ratio;
        d.alpha[(size_t)s * D + k] = al;
        p_part += (al * al + il) * d.phi_c[k];
        l_part += log(il);
        i_part += il;
        a_part += al * al;
    }
    // four block sums: a fixed shuffle tree inside each warp, then the warps' partials in warp order
    double parts[4] = {p_part, l_part, i_part, a_part};
    __syncthreads();   // every thread has read scal[0] (ps)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) parts[q] += __shfl_xor_sync(0xffffffffu, parts[q], o);
        if ((tid & 31) == 0) red[q * (kEThreads / 32) + (tid >> 5)] = parts[q];
    }
    __syncthreads();
    if (tid < 4) {
        double acc = 0.0;
        for (int w = 0; w < kEThreads / 32; ++w) acc += red[tid * (kEThreads / 32) + w];
        scal[tid] = acc;
    }
    __syncthreads();
    if (tid == 0) {
        d.phiTerm[s] = scal[0];
        d.logPi[s] = log(fmax(pi_s, 1e-8));
        d.fsums[cur][3 * s] = scal[1];
        d.fsums[cur][3 * s + 1] = scal[2];
        d.fsums[cur][3 * s + 2] = scal[3];
    }
}

// use_tile: the block's rho [D x 128 frames] is staged in shared memory once (coalesced, every load in flight at once) and
// feeds both the E-step and the partial sums: the per-thread chains then wait on shared memory, not on L2.
__global__ void __launch_bounds__(kEThreads) vbx_estep_kernel2(Dev d, int use_tile) {
    if (d.state[0]) return;
    extern __shared__ double sm[];
    const int S = d.S, D = d.D, tid = threadIdx.x, b = blockIdx.x;
    double *a_s = sm;                        // [S x D] alpha
    double *off_s = a_s + (size_t)S * D;     // [S] -0.5 phi
    double *lpi_s = off_s + S;               // [S]
    double *g_s = lpi_s + S;                 // [kEThreads x S] this block's new gamma rows
    double *red = g_s + (size_t)kEThreads * S;   // [kEThreads]
    double *tile = use_tile ? red + kEThreads : nullptr;   // [D x (kEThreads + 1)]
    if (use_tile) {
        const int t0 = b * kEThreads;
        for (int i = tid; i < D * kEThreads; i += kEThreads) {
            const int k = i / kEThreads, r = i - k * kEThreads;
            tile[k * (kEThreads + 1) + r] = (t0 + r < d.T) ? d.rhoT[(size_t)k * d.Tp + t0 + r] : 0.0;
        }
    }
    for (int o = tid; o < S * D; o += kEThreads) a_s[o] = d.alpha[o];
    for (int c = tid; c < S; c += kEThreads) {
        off_s[c] = d.phiTerm[c] * -0.5;
        lpi_s[c] = d.logPi[c];
    }
    __syncthreads();
    const int t0 = b * kEThreads, rows = min(kEThreads, d.T - t0), t = t0 + tid;
    double ll = 0.0;
    if (t < d.T) {
        double *g = g_s + (size_t)tid * S;
        const double Gt = d.G[t];
        const double *xr = d.rhoT + t;
        double mx = -1.7976931348623157e308;
        for (int s0 = 0; s0 < S; s0 += kSG) {
            double acc[kSG];
#pragma unroll
            for (int q = 0; q < kSG; ++q) acc[q] = 0.0;
            for (int k = 0; k < D; ++k) {
                const double x = tile ? tile[k * (kEThreads + 1) + tid] : xr[(size_t)k * d.Tp];
#pragma unroll
                for (int q = 0; q < kSG; ++q)
                    if (s0 + q < S) acc[q] += x * a_s[(size_t)(s0 + q) * D + k];
            }
#pragma unroll
            for (int q = 0; q < kSG; ++q)
                if (s0 + q < S) {
                    const double v = ((acc[q] + off_s[s0 + q]) + Gt) * d.Fa + lpi_s[s0 + q];
                    g[s0 + q] = v;
                    mx = fmax(mx, v);
                }
        }
        double sum = 0.0;
        for (int c = 0; c < S; ++c) {
            const double e = exp(g[c] - mx);
            g[c] = e;
            sum += e;
        }
        if (sum <= 0.0 || !isfinite(sum)) {
            for (int c = 0; c < S; ++c) g[c] = 1.0 / (double)S;
            ll = mx;
        } else {
            const double inv = 1.0 / sum;
            for (int c = 0; c < S; ++c) g[c] *= inv;
            ll = mx + log(sum);
        }
        double *gout = d.gamma + (size_t)t * S;
        for (int c = 0; c < S; ++c) gout[c] = g[c];
    }
    red[tid] = ll;
    __syncthreads();
    if (tid == 0) {
        double acc = 0.0;
        for (int i = 0; i < kEThreads; ++i) acc += red[i];
        d.fLL[b] = acc;
    }
    vbx_block_partials(d, g_s, t0, rows, b, tile);
}

// first maximum wins (VBxClustering.swift:144-146)
__global__ void vbx_hard_kernel(const double *__restrict__ gamma, int T, int S, int *__restrict__ hard) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const double *g = gamma + (size_t)t * S;
    int best = 0;
    for (int s = 1; s < S; ++s)
        if (g[best] < g[s]) best = s;
    hard[t] = best;
}

// ---- centroids ----------------------------------------------------------------------------------------
// per chunk: num[c][s][k] = sum_t (gamma>0) gamma[t][s] e[t][k], den[c][s] = sum_t gamma   (:642-674)
__global__ void centroid_accumulate_kernel(const double *__restrict__ emb, const double *__restrict__ gamma, int T,
                                           int E, int S, int chunks, double *__restrict__ pnum,
                                           double *__restrict__ pden) {
    const int c = blockIdx.x;
    const int per = (T + chunks - 1) / chunks;
    const int t0 = c * per, t1 = min(T, t0 + per);
    const int SE = S * E;
    for (int o = threadIdx.x; o < SE; o += blockDim.x) {
        const int s = o / E, k = o % E;
        double acc = 0.0;
        for (int t = t0; t < t1; ++t) {
            const double w = gamma[(size_t)t * S + s];
            if (w > 0.0) acc += w * emb[(size_t)t * E + k];
        }
        pnum[(size_t)c * SE + o] = acc;
    }
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        double acc = 0.0;
        for (int t = t0; t < t1; ++t) {
            const double w = gamma[(size_t)t * S + s];
            if (w > 0.0) acc += w;
        }
        pden[(size_t)c * S + s] = acc;
    }
}

// single CTA: speakers with pi > 1e-7 in ascending order become centroids 0..K-1; also L2-normalised copies
__global__ void centroid_finish_kernel(const double *__restrict__ pnum, const double *__restrict__ pden,
                                       const double *__restrict__ pi, int E, int S, int chunks, int *__restrict__ map,
                                       double *__restrict__ cent, double *__restrict__ cent_n, int *__restrict__ count) {
    __shared__ int K;
    if (threadIdx.x == 0) {
        int k = 0;
        for (int s = 0; s < S; ++s) map[s] = (pi[s] > 1e-7) ? k++ : -1;
        K = k;
        *count = k;
    }
    __syncthreads();
    for (int o = threadIdx.x; o < S * E; o += blockDim.x) {
        const int s = o / E, k = o % E;
        if (map[s] < 0) continue;
        double num = 0.0, den = 0.0;
        for (int c = 0; c < chunks; ++c) {
            num += pnum[(size_t)c * S * E + o];
            den += pden[(size_t)c * S + s];
        }
        cent[(size_t)map[s] * E + k] = den > 0.0 ? num / den : 0.0;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < K; c += blockDim.x) {   // normalize (:824-860): unchanged if |c|^2 <= 0
        const double *v = cent + (size_t)c * E;
        double ss = 0.0;   // individually rounded operations, like the reference's scalar loops (no FMA contraction)
        for (int k = 0; k < E; ++k) ss = __dadd_rn(ss, __dmul_rn(v[k], v[k]));
        const double sc = ss > 0.0 ? __ddiv_rn(1.0, __dsqrt_rn(ss)) : 1.0;
        for (int k = 0; k < E; ++k) cent_n[(size_t)c * E + k] = __dmul_rn(v[k], sc);
    }
}

// ---- centroids, parallel path (S <= kFusedMaxS): the same sums over kFChunks chunks, thread per (s, k) and chunk; the
// fold over chunks and the division run thread-per-output on many CTAs, the normalisation thread-per-centroid.
// per block of kCBlock frames: num[b][s][k] = sum_t (gamma > 0) gamma[t][s] e[t][k] (thread per dimension k, eight speakers
// at a time in registers: one embedding load feeds eight predicated FMAs), den[b][s] = sum_t gamma   (:642-674)
constexpr int kCBlock = 128;
__global__ void __launch_bounds__(256) centroid_acc16_kernel(const double *__restrict__ emb, const double *__restrict__ gamma,
                                                             int T, int E, int S, double *__restrict__ pnum,
                                                             double *__restrict__ pden) {
    extern __shared__ double g_s[];   // [kCBlock x S] this block's gamma rows
    const int b = blockIdx.x, t0 = b * kCBlock, rows = min(kCBlock, T - t0);
    for (int i = threadIdx.x; i < rows * S; i += 256) g_s[i] = gamma[(size_t)t0 * S + i];
    __syncthreads();
    for (int s = threadIdx.x; s < S; s += 256) {
        double acc = 0.0;
        for (int r = 0; r < rows; ++r) {
            const double w = g_s[r * S + s];
            if (w > 0.0) acc += w;
        }
        pden[(size_t)b * S + s] = acc;
    }
    for (int k = threadIdx.x; k < E; k += 256) {
        const double *ek = emb + (size_t)t0 * E + k;
        for (int s0 = 0; s0 < S; s0 += kSG) {
            double acc[kSG];
#pragma unroll
            for (int q = 0; q < kSG; ++q) acc[q] = 0.0;
            for (int r = 0; r < rows; ++r) {
                const double x = ek[(size_t)r * E];
                const double *g = g_s + r * S + s0;
#pragma unroll
                for (int q = 0; q < kSG; ++q)
                    if (s0 + q < S) {
                        const double w = g[q];
                        if (w > 0.0) acc[q] += w * x;
                    }
            }
#pragma unroll
            for (int q = 0; q < kSG; ++q)
                if (s0 + q < S) pnum[((size_t)b * S + s0 + q) * E + k] = acc[q];
        }
    }
}
__global__ void __launch_bounds__(256) centroid_fold_kernel(const double *__restrict__ pnum, const double *__restrict__ pden,
                                                            const double *__restrict__ pi, int E, int S, int blocks,
                                                            double *__restrict__ cent) {
    const int o = blockIdx.x * 256 + threadIdx.x;
    if (o >= S * E) return;
    const int s = o / E;
    if (!(pi[s] > 1e-7)) return;
    int slot = 0;
    for (int j = 0; j < s; ++j) slot += pi[j] > 1e-7 ? 1 : 0;
    double num = 0.0, den = 0.0;
#pragma unroll 8
    for (int b = 0; b < blocks; ++b) {   // blocks ascending
        num += pnum[(size_t)b * S * E + o];
        den += pden[(size_t)b * S + s];
    }
    cent[(size_t)slot * E + (o - s * E)] = den > 0.0 ? num / den : 0.0;
}
__global__ void centroid_norm_kernel(const double *__restrict__ pi, int E, int S, const double *__restrict__ cent,
                                     double *__restrict__ cent_n, int *__restrict__ count) {
    int K = 0;
    for (int s = 0; s < S; ++s) K += pi[s] > 1e-7 ? 1 : 0;
    if (threadIdx.x == 0) *count = K;
    for (int c = threadIdx.x; c < K; c += blockDim.x) {   // normalize (:824-860): unchanged if |c|^2 <= 0
        const double *v = cent + (size_t)c * E;
        double ss = 0.0;
        for (int k = 0; k < E; ++k) ss = __dadd_rn(ss, __dmul_rn(v[k], v[k]));
        const double sc = ss > 0.0 ? __ddiv_rn(1.0, __dsqrt_rn(ss)) : 1.0;
        for (int k = 0; k < E; ++k) cent_n[(size_t)c * E + k] = __dmul_rn(v[k], sc);
    }
}

// thread per embedding: cosine against every centroid, strict '>' (OfflineDiarizerManager.swift:800-822), scores optional
// [N x K].  Tiled: 128 embeddings per CTA, 32 dimensions at a time through a padded shared-memory tile so that
// the row-major embeddings are read coalesced; eight centroids per pass share one sweep over the row.  Per (n, c) the
// arithmetic is the reference's scalar loop (individually rounded operations, k ascending): exact ties resolve the same way.
constexpr int kATile = 32, kARows = 128, kAGroup = 8;
__global__ void __launch_bounds__(kARows) assign_tiled_kernel(const double *__restrict__ emb, int N, int E,
                                                              const double *__restrict__ cent_n,
                                                              const int *__restrict__ count_ptr, int K_fixed,
                                                              int *__restrict__ labels, double *__restrict__ scores) {
    __shared__ double tile[kARows][kATile + 1];
    const int K = count_ptr ? *count_ptr : K_fixed;
    const int n0 = blockIdx.x * kARows, r = threadIdx.x, n = n0 + r;
    if (K <= 0) {
        if (n < N) labels[n] = 0;
        return;
    }
    auto load_tile = [&](int k0) {
        __syncthreads();
        for (int idx = threadIdx.x; idx < kARows * kATile; idx += kARows) {
            const int rr = idx / kATile, j = idx - rr * kATile;
            tile[rr][j] = (n0 + rr < N && k0 + j < E) ? emb[(size_t)(n0 + rr) * E + k0 + j] : 0.0;
        }
        __syncthreads();
    };
    double ss = 0.0;
    for (int k0 = 0; k0 < E; k0 += kATile) {
        load_tile(k0);
        const int lim = min(kATile, E - k0);
        for (int j = 0; j < lim; ++j) ss = __dadd_rn(ss, __dmul_rn(tile[r][j], tile[r][j]));
    }
    const double sc = ss > 0.0 ? __ddiv_rn(1.0, __dsqrt_rn(ss)) : 1.0;
    int best = 0;
    double best_score = -INFINITY;
    for (int c0 = 0; c0 < K; c0 += kAGroup) {
        const int gc = min(kAGroup, K - c0);
        double dot[kAGroup];
#pragma unroll
        for (int q = 0; q < kAGroup; ++q) dot[q] = 0.0;
        for (int k0 = 0; k0 < E; k0 += kATile) {
            load_tile(k0);
            const int lim = min(kATile, E - k0);
            for (int j = 0; j < lim; ++j) {
                const double ek = __dmul_rn(tile[r][j], sc);
#pragma unroll
                for (int q = 0; q < kAGroup; ++q)
                    if (q < gc) dot[q] = __dadd_rn(dot[q], __dmul_rn(ek, __ldg(cent_n + (size_t)(c0 + q) * E + k0 + j)));
            }
        }
        if (n < N) {
#pragma unroll
            for (int q = 0; q < kAGroup; ++q) {
                if (q >= gc) break;
                if (scores) scores[(size_t)n * K + c0 + q] = dot[q];
                if (dot[q] > best_score) {
                    best_score = dot[q];
                    best = c0 + q;
                }
            }
        }
    }
    if (n < N) labels[n] = best;
}

__global__ void finite_rows_kernel(const float *__restrict__ emb, int N, int E, unsigned char *__restrict__ ok) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    bool fin = true;
    for (int k = 0; k < E; ++k) fin = fin && isfinite(emb[(size_t)n * E + k]);
    ok[n] = fin ? 1 : 0;
}

__global__ void gather_rows_kernel(const double *__restrict__ src, const int *__restrict__ idx, int rows, int dim,
                                   double *__restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)rows * dim) return;
    const int r = (int)(i / dim), k = (int)(i % dim);
    dst[i] = src[(size_t)idx[r] * dim + k];
}

// ------------------------------------------------------------------------------------------------ host side
static size_t fused_smem_bytes(int S, int D) {
    return sizeof(double) * ((size_t)S * D + 2 * (size_t)S + (size_t)kEThreads * S + kEThreads);
}
static bool fused_path(int S, int D) { return S <= kFusedMaxS && fused_smem_bytes(S, D) <= 200 * 1024; }

int set_smem_limits() {
    FA_CUDA_TRY(cudaFuncSetAttribute(vbx_estep_kernel2, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FA_CUDA_TRY(cudaFuncSetAttribute(vbx_partials0_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FA_CUDA_TRY(cudaFuncSetAttribute(vbx_estep_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    FA_CUDA_TRY(cudaFuncSetAttribute(centroid_acc16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(sizeof(double) * kCBlock * kFusedMaxS)));
    return FA_OK;
}

// d_x: [T x D] device, h_psi: [D] HOST (already identity-substituted by the caller if lengths mismatch),
// d_init: [T] device labels (or nullptr), d_gamma [T x S], d_pi [S], d_elbos [max(max_it,1)], d_hard [T].
int refine_device(DeviceBuffer<> &pool, const double *d_x, int T, int D, const double *h_psi, const int *d_init, int S,
                  const Config &cfg, double *d_gamma, double *d_pi, double *d_elbos, int *d_hard, int *iterations_host,
                  cudaStream_t stream) {
    if (T <= 0 || D <= 0 || S <= 0) return FA_INVALID_ARGUMENT;
    const int max_it = cfg.max_iterations;
    Dev d{};
    d.T = T;
    d.D = D;
    d.S = S;
    d.Tp = (T + 31) & ~31;
    d.chunks = chunks_for(S);
    d.eblocks = (T + kEThreads - 1) / kEThreads;
    d.x = d_x;
    double *phi_c = nullptr;
    int st = carve_arena(pool, [&](Carver &c) {
        d.rho = c.take<double>((size_t)T * D);
        d.rhoT = c.take<double>((size_t)D * d.Tp);
        d.G = c.take<double>(T);
        phi_c = c.take<double>(D);
        d.invL = c.take<double>((size_t)S * D);
        d.alpha = c.take<double>((size_t)S * D);
        d.phiTerm = c.take<double>(S);
        d.logPi = c.take<double>(S);
        d.gsum = c.take<double>(S);
        d.pA = c.take<double>((size_t)d.chunks * S * D);
        d.pG = c.take<double>((size_t)d.chunks * S);
        d.pLL = c.take<double>(d.eblocks);
        d.pPi = c.take<double>((size_t)d.eblocks * S);
        (void)c.take<double>(std::max(max_it, 1));
        d.scal = c.take<double>(8);
        d.state = c.take<int>(8);
        if (S <= kFusedMaxS) {
            d.fA = c.take<double>((size_t)d.eblocks * S * D);
            d.fG = c.take<double>((size_t)d.eblocks * S);
            d.fLL = c.take<double>(d.eblocks);
            for (int i = 0; i < 2; ++i) d.fsums[i] = c.take<double>(3 * (size_t)S);
        }
    }, 512);
    if (st != FA_OK) return st;
    d.phi_c = phi_c;
    d.gamma = d_gamma;
    d.pi = d_pi;
    d.elbos = d_elbos;
    d.Fa = cfg.Fa;
    d.Fb = cfg.Fb;
    d.eps = cfg.epsilon;

    // phi clamp (:239) and pi = 1/S (:237) via tiny host staging
    std::vector<double> h_pi(S, 1.0 / (double)S), h_scal(8, 0.0);
    h_scal[3] = -1.7976931348623157e308;
    FA_CUDA_TRY(cudaMemcpyAsync(d_pi, h_pi.data(), S * sizeof(double), cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaMemcpyAsync(d.scal, h_scal.data(), 8 * sizeof(double), cudaMemcpyHostToDevice, stream));
    FA_CUDA_TRY(cudaMemsetAsync(d.state, 0, 8 * sizeof(int), stream));
    FA_CUDA_TRY(cudaMemsetAsync(d_elbos, 0, std::max(max_it, 1) * sizeof(double), stream));
    {
        std::vector<double> tmp(D);
        for (int k = 0; k < D; ++k) tmp[k] = std::max(h_psi[k], 1e-12);
        FA_CUDA_TRY(cudaMemcpyAsync(phi_c, tmp.data(), D * sizeof(double), cudaMemcpyHostToDevice, stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));   // tmp, h_pi and h_scal are pageable stack/heap buffers
    }
    FA_CUDA_TRY(fa::launch(vbx_init_kernel, (T + 127) / 128, 128, 0, stream, d, d_init, cfg.init_smoothing));
    if (fused_path(S, D)) {
        const size_t tile_bytes = sizeof(double) * (size_t)D * (kEThreads + 1);
        const bool use_tile = fused_smem_bytes(S, D) + tile_bytes <= 200 * 1024;
        const size_t fsmem = fused_smem_bytes(S, D) + (use_tile ? tile_bytes : 0);
        FA_CUDA_TRY(fa::launch(vbx_partials0_kernel, d.eblocks, kEThreads, sizeof(double) * (size_t)kEThreads * S, stream, d));
        for (int it = 0; it < max_it; ++it) {
            FA_CUDA_TRY(fa::launch(vbx_update_kernel2, S, kEThreads, 0, stream, d, it, 0));
            FA_CUDA_TRY(fa::launch(vbx_estep_kernel2, d.eblocks, kEThreads, fsmem, stream, d, use_tile ? 1 : 0));
        }
        if (max_it > 0)   // books of the last E-step (no-op if converged)
            FA_CUDA_TRY(fa::launch(vbx_update_kernel2, S, kEThreads, 0, stream, d, max_it, 1));
    } else {
        const size_t esmem_full = sizeof(double) * ((size_t)S * D + 2 * S + kEThreads);
        const bool alpha_smem = esmem_full <= 200 * 1024;
        const size_t esmem = alpha_smem ? esmem_full : sizeof(double) * kEThreads;
        for (int it = 0; it < max_it; ++it) {
            FA_CUDA_TRY(fa::launch(vbx_accumulate_kernel, d.chunks, 256, 0, stream, d));
            FA_CUDA_TRY(fa::launch(vbx_update_kernel, 1, 256, 0, stream, d));
            FA_CUDA_TRY(fa::launch(alpha_smem ? vbx_estep_kernel<true> : vbx_estep_kernel<false>, d.eblocks, kEThreads, esmem,
                                   stream, d));
            FA_CUDA_TRY(fa::launch(vbx_finish_kernel, 1, 256, 0, stream, d, it));
        }
    }
    FA_CUDA_TRY(fa::launch(vbx_hard_kernel, (T + 127) / 128, 128, 0, stream, d_gamma, T, S, d_hard));
    if (iterations_host) {
        int h_state[2] = {0, 0};
        FA_CUDA_TRY(cudaMemcpyAsync(h_state, d.state, 2 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        FA_CUDA_TRY(cudaStreamSynchronize(stream));
        *iterations_host = h_state[1];
    }
    return FA_OK;
}

int centroids_device(DeviceBuffer<> &pool, const double *d_emb, int T, int E, const double *d_gamma, const double *d_pi,
                     int S, double *d_cent, double *d_cent_n, int *d_count, cudaStream_t stream) {
    const int chunks = S <= kFusedMaxS ? (T + kCBlock - 1) / kCBlock : chunks_for(S);
    double *pnum = nullptr, *pden = nullptr;
    int *map = nullptr;
    int st = carve_arena(pool, [&](Carver &c) {
        pnum = c.take<double>((size_t)chunks * S * E);
        pden = c.take<double>((size_t)chunks * S);
        map = c.take<int>(S);
    }, 2048);
    if (st != FA_OK) return st;
    if (S <= kFusedMaxS) {
        const unsigned tiles = (unsigned)((S * E + 255) / 256);
        FA_CUDA_TRY(fa::launch(centroid_acc16_kernel, chunks, 256, sizeof(double) * (size_t)kCBlock * S, stream, d_emb, d_gamma,
                               T, E, S, pnum, pden));
        FA_CUDA_TRY(fa::launch(centroid_fold_kernel, tiles, 256, 0, stream, pnum, pden, d_pi, E, S, chunks, d_cent));
        FA_CUDA_TRY(fa::launch(centroid_norm_kernel, 1, 64, 0, stream, d_pi, E, S, d_cent, d_cent_n, d_count));
        return FA_OK;
    }
    FA_CUDA_TRY(fa::launch(centroid_accumulate_kernel, chunks, 256, 0, stream, d_emb, d_gamma, T, E, S, chunks, pnum, pden));
    FA_CUDA_TRY(fa::launch(centroid_finish_kernel, 1, 256, 0, stream, pnum, pden, d_pi, E, S, chunks, map, d_cent, d_cent_n,
                           d_count));
    return FA_OK;
}

int assign_device(const double *d_emb, int N, int E, const double *d_cent_n, const int *d_count, int K_fixed,
                  int *d_labels, double *d_scores, cudaStream_t stream) {
    if (N <= 0) return FA_OK;
    FA_CUDA_TRY(fa::launch(assign_tiled_kernel, (N + kARows - 1) / kARows, kARows, 0, stream, d_emb, N, E, d_cent_n, d_count,
                           K_fixed, d_labels, d_scores));
    return FA_OK;
}

int finite_rows_device(const float *d_emb, int N, int E, unsigned char *d_ok, cudaStream_t stream) {
    FA_CUDA_TRY(fa::launch(finite_rows_kernel, (N + 127) / 128, 128, 0, stream, d_emb, N, E, d_ok));
    return FA_OK;
}

int gather_rows_device(const double *d_src, const int *d_idx, int rows, int dim, double *d_dst, cudaStream_t stream) {
    const long long total = (long long)rows * dim;
    if (total <= 0) return FA_OK;
    FA_CUDA_TRY(fa::launch(gather_rows_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, d_src, d_idx, rows, dim, d_dst));
    return FA_OK;
}

} // namespace vbx
} // namespace fa
