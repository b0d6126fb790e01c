// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// CPU restatement (plain C++, single thread, IEEE double, no FMA contraction: build with
// -ffp-contract=off) of FluidAudio's offline clustering backend.  Only tests/, smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library.
//
// Follows:
//   A2  Sources/FluidAudio/Diarizer/Offline/Clustering/AHCClustering.swift:70-105   normalizeFeatures
//   A3  Sources/FastClusterWrapper/FastClusterWrapper.cpp:26-147,196-244 + fastcluster_internal.hpp:1625-1800
//       (generic_linkage_vector_alternative<METHOD_VECTOR_CENTROID>), heap :778-937, list :299-350
//   A5  FastClusterWrapper.cpp:149-192  SciPy-format rows
//   A6  AHCClustering.swift:112-121,124-197  clampDistanceThreshold + assignmentsFromDendrogram
//   A7  AHCClustering.swift:200-210  remapClusterIds
//   V1/V2 Sources/FluidAudio/Diarizer/Offline/Clustering/VBxClustering.swift:41-165,167-664
//   P2  Sources/FluidAudio/Diarizer/Offline/Core/OfflineDiarizerManager.swift:613-691 computeCentroids
//   P3  OfflineDiarizerManager.swift:789-883 centroidScores / assignEmbeddings / normalize / dot
//
// Parity status:
//   * A3 is PINNED: oracle/_ref/liboracle_fc.so is the unmodified reference C++ compiled here; tests require
//     this restatement to reproduce its dendrogram bit for bit (ids and IEEE doubles) on random, clustered,
//     duplicate-heavy and lattice inputs.
//   * A1/A6/A7 are pinned at label level by the reference's own unit tests (AHCClusteringTests.swift).
//   * V1/V2/P2/P3: "parity unpinned" beyond this restatement — no reference test executes VBx and its BLAS /
//     vForce calls are closed-source Accelerate (summation order unknown).  Sums here are sequential in index
//     order; hard labels are the contract.

#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>
#include <algorithm>

namespace {

// ---- indexed binary min-heap with the exact sift rules of fastcluster_internal.hpp:778-937 -------------
// Keys live in an external array `key`; `at[pos]` is the element at heap position pos and `where[elem]`
// its inverse.  Tie behaviour (strict '<' when sifting up, '>=' tests when sifting down, left child first)
// is what decides which of several equal-distance pairs merges first, so it is restated exactly.
struct NNHeap {
    double *key;
    int size;
    std::vector<int> at, where;
    NNHeap(double *key_, int count, int universe, int first) : key(key_), size(count), at(count), where(universe) {
        for (int i = 0; i < count; ++i) {
            where[i + first] = i;
            at[i] = i + first;
        }
    }
    double val(int pos) const { return key[at[pos]]; }
    void swap_pos(int a, int b) {
        std::swap(at[a], at[b]);
        where[at[a]] = a;
        where[at[b]] = b;
    }
    void sift_up(int pos) {
        while (pos > 0) {
            const int parent = (pos - 1) >> 1;
            if (!(val(pos) < val(parent))) break;
            swap_pos(pos, parent);
            pos = parent;
        }
    }
    void sift_down(int pos) {
        for (;;) {
            int child = 2 * pos + 1;
            if (child >= size) break;
            if (val(child) >= val(pos)) {
                ++child;
                if (child >= size || val(child) >= val(pos)) break;
            } else if (child + 1 < size && val(child + 1) < val(child)) {
                ++child;
            }
            swap_pos(pos, child);
            pos = child;
        }
    }
    void heapify() {
        for (int pos = size >> 1; pos > 0;) {
            --pos;
            sift_down(pos);
        }
    }
    int top() const { return at[0]; }
    void raise_key(int elem, double v) {  // new value >= old
        key[elem] = v;
        sift_down(where[elem]);
    }
    void lower_key(int elem, double v) {  // new value <= old
        key[elem] = v;
        sift_up(where[elem]);
    }
    void erase(int elem) {
        --size;
        const int pos = where[elem];
        where[at[size]] = pos;
        at[pos] = at[size];
        if (val(size) <= key[elem]) sift_up(pos); else sift_down(pos);
    }
    void rename(int old_elem, int new_elem, double v) {
        where[new_elem] = where[old_elem];
        at[where[new_elem]] = new_elem;
        if (v <= key[old_elem]) lower_key(new_elem, v); else raise_key(new_elem, v);
    }
};

// ascending list of live node ids with O(1) removal (fastcluster_internal.hpp:299-350)
struct LiveList {
    int head = 0;
    std::vector<int> next, prev;
    explicit LiveList(int n) : next(n + 1), prev(n + 1) {
        for (int i = 0; i < n; ++i) {
            prev[i + 1] = i;
            next[i] = i + 1;
        }
    }
    void drop(int id) {
        if (id == head) head = next[id];
        else {
            next[prev[id]] = next[id];
            prev[next[id]] = prev[id];
        }
        next[id] = 0;
    }
    bool dead(int id) const { return next[id] == 0; }
};

struct NanFound {};

} // namespace

extern "C" {

// A2: row-wise L2 normalisation, scale = norm>0 ? 1/sqrt(sum x^2) : 0
void oracle_l2_normalize_rows(const double *x, int64_t n, int64_t d, double *out) {
    for (int64_t r = 0; r < n; ++r) {
        double s = 0;
        for (int64_t k = 0; k < d; ++k) s += x[r * d + k] * x[r * d + k];
        const double scale = s > 0 ? 1.0 / std::sqrt(s) : 0.0;
        for (int64_t k = 0; k < d; ++k) out[r * d + k] = x[r * d + k] * scale;
    }
}

// A3+A5: same status codes as FastClusterWrapper.h:11-19
int32_t oracle_centroid_linkage(const double *data, uint64_t point_count, uint64_t dimension, double *Z,
                                uint64_t z_len) {
    if (!data || !Z) return 1;
    if (point_count == 0) return 0;
    if (dimension == 0) return 1;
    if (point_count > 0x7fffffffull || dimension > 0x7fffffffull) return 2;
    const uint64_t need = point_count > 1 ? (point_count - 1) * 4 : 0;
    if (z_len < need) return 3;
    if (point_count == 1) return 0;
    try {
        const int N = (int)point_count, D = (int)dimension;
        std::vector<double> merged((size_t)(N - 1) * D);
        std::vector<int> weight(2 * N - 1, 0);
        for (int i = 0; i < N; ++i) weight[i] = 1;
        auto vec = [&](int id) -> const double * {
            return id < N ? data + (size_t)id * D : merged.data() + (size_t)(id - N) * D;
        };
        auto sqdist = [&](int a, int b) -> double {
            const double *pa = vec(a), *pb = vec(b);
            double s = 0;
            for (int k = 0; k < D; ++k) {
                const double diff = pa[k] - pb[k];
                s += diff * diff;
            }
            if (s != s) throw NanFound();
            return s;
        };
        std::vector<int> nn(2 * N - 2);
        std::vector<double> nnd(2 * N - 2);
        LiveList live(2 * N - 1);
        NNHeap heap(nnd.data(), N - 1, 2 * N - 2, 1);
        std::vector<int> ma(N - 1), mb(N - 1);
        std::vector<double> md(N - 1);

        for (int i = 1; i < N; ++i) {
            double best = std::numeric_limits<double>::infinity();
            int arg = 0;
            for (int j = 0; j < i; ++j) {
                const double t = sqdist(i, j);
                if (t < best) {
                    best = t;
                    arg = j;
                }
            }
            nnd[i] = best;
            nn[i] = arg;
        }
        heap.heapify();
        for (int step = 0; step < N - 1; ++step) {
            const int fresh = N + step;
            int a = heap.top();
            while (live.dead(nn[a])) {
                int j = live.head;
                nn[a] = j;
                double best = sqdist(a, j);
                for (j = live.next[j]; j < a; j = live.next[j]) {
                    const double t = sqdist(a, j);
                    if (t < best) {
                        best = t;
                        nn[a] = j;
                    }
                }
                heap.raise_key(a, best);
                a = heap.top();
            }
            const int b = nn[a];
            live.drop(a);
            live.drop(b);
            ma[step] = a;
            mb[step] = b;
            md[step] = nnd[a];
            if (step < N - 2) {
                double *pn = merged.data() + (size_t)step * D;
                const double *pa = vec(a), *pb = vec(b);
                const double wa = (double)weight[a], wb = (double)weight[b];
                const double den = wa + wb;
                for (int k = 0; k < D; ++k) pn[k] = (pa[k] * wa + pb[k] * wb) / den;
                weight[fresh] = weight[a] + weight[b];
                int j = live.head;
                nn[fresh] = j;
                double best = sqdist(j, fresh);
                for (j = live.next[j]; j < fresh; j = live.next[j]) {
                    const double t = sqdist(j, fresh);
                    if (t < best) {
                        best = t;
                        nn[fresh] = j;
                    }
                }
                if (b < live.head) heap.erase(live.head); else heap.erase(b);
                heap.rename(a, fresh, best);
            }
        }
        // postprocess: sqrt of every merge distance, then SciPy rows (min id, max id, dist, size)
        for (int s = 0; s < N - 1; ++s) {
            const int lo = std::min(ma[s], mb[s]), hi = std::max(ma[s], mb[s]);
            const double sz = (lo < N ? 1.0 : Z[(size_t)(lo - N) * 4 + 3]) + (hi < N ? 1.0 : Z[(size_t)(hi - N) * 4 + 3]);
            Z[(size_t)s * 4 + 0] = (double)lo;
            Z[(size_t)s * 4 + 1] = (double)hi;
            Z[(size_t)s * 4 + 2] = std::sqrt(md[s]);
            Z[(size_t)s * 4 + 3] = sz;
        }
        return 0;
    } catch (const std::bad_alloc &) {
        return 4;
    } catch (const NanFound &) {
        return 5;
    } catch (...) {
        return 255;
    }
}

// A6 + A7: threshold clamp, top-down cut using each node's own merge distance, relabel by first appearance.
void oracle_dendrogram_cut(const double *Z, int64_t count, double threshold, int32_t *labels) {
    if (count <= 0) return;
    if (count == 1) {
        labels[0] = 0;
        return;
    }
    double thr;
    if (threshold != threshold) thr = 0;
    else thr = std::max(0.0, std::min(2.0, threshold));
    const int64_t total = 2 * count - 1;
    std::vector<int64_t> left(total, -1), right(total, -1);
    std::vector<double> dist(total, 0.0);
    for (int64_t m = 0; m < count - 1; ++m) {
        left[count + m] = (int64_t)Z[m * 4];
        right[count + m] = (int64_t)Z[m * 4 + 1];
        dist[count + m] = Z[m * 4 + 2];
    }
    std::vector<int64_t> assign(count, -1), stack{total - 1}, queue;
    int64_t next_label = 0;
    while (!stack.empty()) {
        const int64_t node = stack.back();
        stack.pop_back();
        if (node < 0) continue;
        if (node < count) {
            if (assign[node] == -1) assign[node] = next_label++;
            continue;
        }
        if (dist[node] <= thr) {
            const int64_t label = next_label++;
            queue.assign(1, node);
            while (!queue.empty()) {
                const int64_t cur = queue.back();
                queue.pop_back();
                if (cur < count) assign[cur] = label;
                else {
                    if (left[cur] >= 0) queue.push_back(left[cur]);
                    if (right[cur] >= 0) queue.push_back(right[cur]);
                }
            }
        } else {
            if (left[node] >= 0) stack.push_back(left[node]);
            if (right[node] >= 0) stack.push_back(right[node]);
        }
    }
    for (int64_t i = 0; i < count; ++i)
        if (assign[i] == -1) assign[i] = next_label++;
    // remapClusterIds
    std::vector<int64_t> map(next_label, -1);
    int64_t next_id = 0;
    for (int64_t i = 0; i < count; ++i) {
        if (map[assign[i]] < 0) map[assign[i]] = next_id++;
        labels[i] = (int32_t)map[assign[i]];
    }
}

struct oracle_vbx_config {
    double Fa;              // 0.07
    double Fb;              // 0.8
    int32_t max_iterations; // 20
    double epsilon;         // 1e-4
    double init_smoothing;  // 7.0
};

// V1+V2.  features: T x D row-major (rho), phi: D (psi), init: T labels (may be null -> uniform gamma).
// gamma out: T x S, pi out: S, elbos out: max(max_iterations,1) capacity, hard: T.
// Returns the number of iterations run; *speakers = S.
int32_t oracle_vbx_refine(const double *features, int64_t T, int64_t D, const double *phi_in, int64_t phi_len,
                          const int32_t *init, const oracle_vbx_config *cfg, int32_t S, double *gamma, double *pi,
                          double *elbos, int32_t *hard) {
    std::vector<double> phi(D);
    if (phi_len != D) std::fill(phi.begin(), phi.end(), 1.0);            // :72-76
    else for (int64_t d = 0; d < D; ++d) phi[d] = phi_in[d];
    // initial gamma (:100-113)
    std::fill(gamma, gamma + T * S, 0.0);
    if (init) {
        for (int64_t t = 0; t < T; ++t) {
            const int32_t sp = std::max(0, std::min(init[t], S - 1));
            gamma[t * S + sp] = 1.0;
        }
    } else {
        for (int64_t i = 0; i < T * S; ++i) gamma[i] = 1.0 / (double)S;
    }
    std::vector<double> row(S);
    if (cfg->init_smoothing >= 0.0) {  // :190-219
        for (int64_t t = 0; t < T; ++t) {
            double *g = gamma + t * S;
            double mx = -std::numeric_limits<double>::max();
            for (int s = 0; s < S; ++s) {
                row[s] = g[s] * cfg->init_smoothing;
                mx = std::max(mx, row[s]);
            }
            double sum = 0;
            for (int s = 0; s < S; ++s) {
                row[s] = std::exp(row[s] - mx);
                sum += row[s];
            }
            if (sum <= 0.0 || !std::isfinite(sum)) for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
            else {
                const double inv = 1.0 / sum;
                for (int s = 0; s < S; ++s) g[s] = row[s] * inv;
            }
        }
    }
    for (int64_t t = 0; t < T; ++t) {  // :221-235
        double *g = gamma + t * S;
        double sum = 0;
        for (int s = 0; s < S; ++s) sum += g[s];
        if (sum <= 0.0 || !std::isfinite(sum)) for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
        else {
            const double inv = 1.0 / sum;
            for (int s = 0; s < S; ++s) g[s] *= inv;
        }
    }
    for (int s = 0; s < S; ++s) pi[s] = 1.0 / (double)S;
    std::vector<double> phic(D), sq(D);
    for (int64_t d = 0; d < D; ++d) {
        phic[d] = std::max(phi[d], 1e-12);
        sq[d] = std::sqrt(phic[d]);
    }
    std::vector<double> rho((size_t)T * D), G(T);
    const double log_const = (double)D * std::log(2.0 * M_PI);
    for (int64_t t = 0; t < T; ++t) {
        double ss = 0;
        for (int64_t d = 0; d < D; ++d) {
            rho[t * D + d] = features[t * D + d] * sq[d];
            ss += features[t * D + d] * features[t * D + d];
        }
        G[t] = -0.5 * (ss + log_const);
    }
    const double ratio = cfg->Fa / cfg->Fb;
    std::vector<double> invL((size_t)S * D), alpha((size_t)S * D), gsum(S), phiTerm(S), logP((size_t)T * S), logPi(S);
    double prev = -std::numeric_limits<double>::max();
    int32_t iterations = 0;
    const int32_t cap = std::max(cfg->max_iterations, 1);
    for (int i = 0; i < cap; ++i) elbos[i] = 0.0;
    for (int32_t it = 0; it < cfg->max_iterations; ++it) {
        iterations = it + 1;
        for (int s = 0; s < S; ++s) gsum[s] = 0;
        for (int64_t t = 0; t < T; ++t)
            for (int s = 0; s < S; ++s) gsum[s] += gamma[t * S + s];
        for (int s = 0; s < S; ++s) {
            const double w = ratio * gsum[s];
            for (int64_t d = 0; d < D; ++d) invL[s * D + d] = 1.0 / std::max(1.0 + w * phic[d], 1e-12);
        }
        // temp = gamma^T rho  (S x D), then alpha = ratio * invL .* temp
        std::fill(alpha.begin(), alpha.end(), 0.0);
        for (int64_t t = 0; t < T; ++t)
            for (int s = 0; s < S; ++s) {
                const double g = gamma[t * S + s];
                for (int64_t d = 0; d < D; ++d) alpha[s * D + d] += g * rho[t * D + d];
            }
        for (size_t i = 0; i < alpha.size(); ++i) alpha[i] = (alpha[i] * invL[i]) * ratio;
        for (int s = 0; s < S; ++s) {
            double sum = 0;
            for (int64_t d = 0; d < D; ++d) sum += (alpha[s * D + d] * alpha[s * D + d] + invL[s * D + d]) * phic[d];
            phiTerm[s] = sum;
        }
        for (int64_t t = 0; t < T; ++t)
            for (int s = 0; s < S; ++s) {
                double acc = 0;
                for (int64_t d = 0; d < D; ++d) acc += rho[t * D + d] * alpha[s * D + d];
                logP[t * S + s] = ((acc + (-0.5 * phiTerm[s])) + G[t]) * cfg->Fa;
            }
        for (int s = 0; s < S; ++s) logPi[s] = std::log(std::max(pi[s], 1e-8));
        double ll = 0;
        for (int64_t t = 0; t < T; ++t) {
            double mx = -std::numeric_limits<double>::max();
            for (int s = 0; s < S; ++s) {
                row[s] = logP[t * S + s] + logPi[s];
                mx = std::max(mx, row[s]);
            }
            double sum = 0;
            for (int s = 0; s < S; ++s) {
                row[s] = std::exp(row[s] - mx);
                sum += row[s];
            }
            double *g = gamma + t * S;
            if (sum <= 0.0 || !std::isfinite(sum)) {
                for (int s = 0; s < S; ++s) g[s] = 1.0 / (double)S;
                ll += mx;
            } else {
                const double inv = 1.0 / sum;
                for (int s = 0; s < S; ++s) g[s] = row[s] * inv;
                ll += mx + std::log(sum);
            }
        }
        for (int s = 0; s < S; ++s) pi[s] = 0;
        for (int64_t t = 0; t < T; ++t)
            for (int s = 0; s < S; ++s) pi[s] += gamma[t * S + s];
        double ps = 0;
        for (int s = 0; s < S; ++s) ps += pi[s];
        if (ps > 0.0 && std::isfinite(ps)) {
            const double inv = 1.0 / ps;
            for (int s = 0; s < S; ++s) pi[s] *= inv;
        } else for (int s = 0; s < S; ++s) pi[s] = 1.0 / (double)S;
        double sLog = 0, sInv = 0, sA2 = 0;
        for (size_t i = 0; i < invL.size(); ++i) {
            sLog += std::log(invL[i]);
            sInv += invL[i];
            sA2 += alpha[i] * alpha[i];
        }
        const double elbo = ll + cfg->Fb * 0.5 * (sLog - sInv - sA2 + (double)invL.size());
        if (it < cap) elbos[it] = elbo;
        if (it > 0 && std::fabs(elbo - prev) < cfg->epsilon) {
            prev = elbo;
            break;
        }
        prev = elbo;
    }
    for (int64_t t = 0; t < T; ++t) {  // first max wins (:144-146)
        int best = 0;
        for (int s = 1; s < S; ++s)
            if (gamma[t * S + best] < gamma[t * S + s]) best = s;
        hard[t] = best;
    }
    return iterations;
}

// P2: gamma/pi weighted centroids over UN-normalised training embeddings, speakers with pi > 1e-7.
// centroids out capacity S x dim.  Returns K (number of centroids); speaker_of[k] = VBx speaker index.
int32_t oracle_compute_centroids(const double *emb, int64_t T, int64_t dim, const double *gamma, const double *pi,
                                 int32_t S, double *centroids, int32_t *speaker_of) {
    int32_t K = 0;
    for (int s = 0; s < S; ++s) {
        if (!(pi[s] > 1e-7)) continue;
        double *c = centroids + (size_t)K * dim;
        for (int64_t k = 0; k < dim; ++k) c[k] = 0;
        double den = 0;
        for (int64_t t = 0; t < T; ++t) {
            const double w = gamma[t * S + s];
            if (!(w > 0)) continue;
            den += w;
            for (int64_t k = 0; k < dim; ++k) c[k] += w * emb[t * dim + k];  // cblas_daxpy
        }
        if (den > 0) for (int64_t k = 0; k < dim; ++k) c[k] /= den;
        else for (int64_t k = 0; k < dim; ++k) c[k] = 0;
        if (speaker_of) speaker_of[K] = s;
        ++K;
    }
    return K;
}

// computeCentroidsFromClusters (:693-746): plain means per distinct label, ordered by label value.
int32_t oracle_centroids_from_clusters(const double *emb, int64_t T, int64_t dim, const int32_t *clusters,
                                       double *centroids, int32_t cap) {
    std::vector<int32_t> keys(clusters, clusters + T);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    if ((int64_t)keys.size() > cap) return -(int32_t)keys.size();
    for (size_t k = 0; k < keys.size(); ++k) {
        double *c = centroids + k * dim;
        for (int64_t j = 0; j < dim; ++j) c[j] = 0;
        int64_t cnt = 0;
        for (int64_t t = 0; t < T; ++t)
            if (clusters[t] == keys[k]) {
                for (int64_t j = 0; j < dim; ++j) c[j] += 1.0 * emb[t * dim + j];
                ++cnt;
            }
        if (cnt > 0) for (int64_t j = 0; j < dim; ++j) c[j] /= (double)cnt;
    }
    return (int32_t)keys.size();
}

// P3: cosine of every embedding vs every centroid, argmax with strict '>' (first max wins).
// scores out (optional): N x K.
void oracle_assign_embeddings(const double *emb, int64_t N, int64_t dim, const double *centroids, int32_t K,
                              int32_t *labels, double *scores) {
    if (K <= 0) {
        for (int64_t i = 0; i < N; ++i) labels[i] = 0;
        return;
    }
    auto normalize = [&](const double *v, double *o) {
        double ss = 0;
        for (int64_t k = 0; k < dim; ++k) ss += v[k] * v[k];
        if (ss <= 0) {
            for (int64_t k = 0; k < dim; ++k) o[k] = v[k];
            return;
        }
        const double sc = 1.0 / std::sqrt(ss);
        for (int64_t k = 0; k < dim; ++k) o[k] = v[k] * sc;
    };
    std::vector<double> cn((size_t)K * dim), en(dim);
    for (int c = 0; c < K; ++c) normalize(centroids + (size_t)c * dim, cn.data() + (size_t)c * dim);
    for (int64_t i = 0; i < N; ++i) {
        normalize(emb + i * dim, en.data());
        int best = 0;
        double best_score = -std::numeric_limits<double>::infinity();
        for (int c = 0; c < K; ++c) {
            double dot = 0;
            for (int64_t k = 0; k < dim; ++k) dot += en[k] * cn[(size_t)c * dim + k];
            if (scores) scores[i * K + c] = dot;
            if (dot > best_score) {
                best_score = dot;
                best = c;
            }
        }
        labels[i] = best;
    }
}

} // extern "C"

// ---- "next" row (SURVEY §8f rank 1): constrained assignment --------------------------------------------------
// P4  Sources/FluidAudio/Diarizer/HungarianAssignment.swift:8-61 (solve), :67-97 (maxScoreAssignment)
//     Sources/FluidAudio/Diarizer/Offline/Clustering/ConstrainedClusterAssignment.swift:20-42 (assign)
//     OfflineDiarizerManager.swift:885-911 (buildChunkAssignments)
// Pinned by the reference's own exact-integer unit tests (HungarianAssignmentTests.swift,
// ConstrainedClusterAssignmentTests.swift), ported in tests/test_oracle_golden.py.
extern "C" {

// Kuhn-Munkres with row/column potentials on a square non-negative integer matrix; assign[row] = col.
void oracle_hungarian_solve(const int64_t *cost, int32_t n, int32_t *assign) {
    if (n <= 0) return;
    const int64_t INF = std::numeric_limits<int64_t>::max() / 4;
    std::vector<int64_t> u(n + 1, 0), v(n + 1, 0), minv(n + 1);
    std::vector<int32_t> p(n + 1, 0), way(n + 1, 0);
    std::vector<char> used(n + 1);
    for (int32_t i = 1; i <= n; ++i) {
        p[0] = i;
        int32_t j0 = 0;
        std::fill(minv.begin(), minv.end(), INF);
        std::fill(used.begin(), used.end(), 0);
        do {
            used[j0] = 1;
            const int32_t i0 = p[j0];
            int64_t delta = INF;
            int32_t j1 = 0;
            for (int32_t j = 1; j <= n; ++j) {
                if (used[j]) continue;
                const int64_t cur = cost[(size_t)(i0 - 1) * n + (j - 1)] - u[i0] - v[j];
                if (cur < minv[j]) {
                    minv[j] = cur;
                    way[j] = j0;
                }
                if (minv[j] < delta) {
                    delta = minv[j];
                    j1 = j;
                }
            }
            for (int32_t j = 0; j <= n; ++j) {
                if (used[j]) {
                    u[p[j]] += delta;
                    v[j] -= delta;
                } else {
                    minv[j] -= delta;
                }
            }
            j0 = j1;
        } while (p[j0] != 0);
        do {
            const int32_t j1 = way[j0];
            p[j0] = p[j1];
            j0 = j1;
        } while (j0 != 0);
    }
    for (int32_t r = 0; r < n; ++r) assign[r] = -1;
    for (int32_t j = 1; j <= n; ++j)
        if (p[j] != 0) assign[p[j] - 1] = j - 1;
}

// scores: rows x cols row-major; assign[row] = col or -1
void oracle_max_score_assignment(const double *scores, int32_t rows, int32_t cols, int32_t *assign) {
    if (rows <= 0) return;
    if (cols <= 0) {
        for (int32_t r = 0; r < rows; ++r) assign[r] = -1;
        return;
    }
    bool any = false;
    double mx = 0, mn = 0;
    for (int64_t i = 0; i < (int64_t)rows * cols; ++i)
        if (std::isfinite(scores[i])) {
            if (!any) mx = mn = scores[i];
            mx = std::max(mx, scores[i]);
            mn = std::min(mn, scores[i]);
            any = true;
        }
    const double sentinel = mn - 1;
    const int32_t n = std::max(rows, cols);
    std::vector<int64_t> cost((size_t)n * n, 0);
    for (int32_t r = 0; r < rows; ++r)
        for (int32_t c = 0; c < cols; ++c) {
            const double s = std::isfinite(scores[(size_t)r * cols + c]) ? scores[(size_t)r * cols + c] : sentinel;
            cost[(size_t)r * n + c] = (int64_t)std::round((mx - s) * 1e6);
        }
    std::vector<int32_t> full(n);
    oracle_hungarian_solve(cost.data(), n, full.data());
    for (int32_t r = 0; r < rows; ++r) assign[r] = full[r] < cols ? full[r] : -1;
}

// scores: N x K; chunk[N]; out[N] = cluster or -2
void oracle_constrained_assign(const double *scores, int64_t N, int32_t K, const int32_t *chunk, int32_t *out) {
    for (int64_t i = 0; i < N; ++i) out[i] = -2;
    std::vector<int64_t> order(N);
    for (int64_t i = 0; i < N; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return chunk[a] < chunk[b]; });
    int64_t i = 0;
    std::vector<double> block;
    std::vector<int32_t> assign;
    while (i < N) {
        int64_t j = i;
        while (j < N && chunk[order[j]] == chunk[order[i]]) ++j;
        const int32_t rows = (int32_t)(j - i);
        block.resize((size_t)rows * std::max(K, 1));
        for (int32_t r = 0; r < rows; ++r)
            for (int32_t c = 0; c < K; ++c) block[(size_t)r * K + c] = scores[order[i + r] * K + c];
        assign.assign(rows, -1);
        oracle_max_score_assignment(block.data(), rows, K, assign.data());
        for (int32_t r = 0; r < rows; ++r) out[order[i + r]] = assign[r] >= 0 ? assign[r] : -2;
        i = j;
    }
}

// matrix [num_chunks x num_speakers], -2 where nothing was assigned
void oracle_build_chunk_assignments(const int32_t *chunk, const int32_t *speaker, const int32_t *assignments, int64_t N,
                                    int32_t num_chunks, int32_t num_speakers, int32_t cluster_count, int32_t *matrix) {
    for (int64_t i = 0; i < (int64_t)num_chunks * num_speakers; ++i) matrix[i] = -2;
    for (int64_t i = 0; i < N; ++i) {
        if (chunk[i] < 0 || chunk[i] >= num_chunks || speaker[i] < 0 || speaker[i] >= num_speakers) continue;
        if (assignments[i] < 0 || assignments[i] >= cluster_count) continue;
        matrix[(int64_t)chunk[i] * num_speakers + speaker[i]] = assignments[i];
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// Speaker-count-constrained re-clustering (SURVEY.md 8f rank 4).
//   KMeansClustering.clusterWithCentroids / clusterWithCentroidsNInit   Diarizer/Offline/Clustering/KMeansClustering.swift:39-130
//   SeededRNG (LCG)                                                     KMeansClustering.swift:212-223
//   SpeakerCountConstraints.resolve / needsAdjustment / targetCount     SpeakerCountConstraints.swift:27-85
// Third-party semantics this depends on and that are NOT in the reference repository: the Swift standard library's
// `MutableCollection.shuffle(using:)`, `Collection.randomElement(using:)`, `Int.random(in:using:)` and
// `RandomNumberGenerator.next(upperBound:)` (swift/stdlib/public/core/{CollectionAlgorithms,Random,Integers}.swift,
// Swift 5.9+/6.x as required by the package's tools version).  Published algorithm, restated here:
//   next(upperBound: u)  -- Lemire's nearly-divisionless method on the full-width product random * u, rejecting while
//                           low < (0 &- u) % u, result = high word;
//   Int.random(in: 0..<n) -- next(upperBound: UInt(n));
//   shuffle               -- for amount = count, count-1, .. 2: swap(current, current + random(0..<amount)), advance;
//   randomElement         -- self[random(0..<count)].
// No Swift toolchain here: this part of the oracle is "parity unpinned" beyond the reference's own seeded
// determinism tests (KMeansClusteringTests.swift), which it satisfies by construction.
struct oracle_lcg {
    uint64_t state;
    uint64_t next() {
        state = state * 6364136223846793005ull + 1442695040888963407ull;
        return state;
    }
    uint64_t next_below(uint64_t upper) {
        unsigned __int128 m = (unsigned __int128)next() * upper;
        if ((uint64_t)m < upper) {
            const uint64_t t = (0 - upper) % upper;
            while ((uint64_t)m < t) m = (unsigned __int128)next() * upper;
        }
        return (uint64_t)(m >> 64);
    }
};

static double oracle_sqdist(const double *a, const double *b, int64_t d) {   // vDSP_vsubD + vDSP_svesqD (:178-185)
    double s = 0.0;
    for (int64_t k = 0; k < d; ++k) {
        const double t = a[k] - b[k];
        s += t * t;
    }
    return s;
}

// normalizeEmbeddings (:133-145): rows with norm <= 1e-10 are kept as they are
void oracle_kmeans_normalize(const double *x, int64_t n, int64_t d, double *out) {
    for (int64_t i = 0; i < n; ++i) {
        double s = 0.0;
        for (int64_t k = 0; k < d; ++k) s += x[i * d + k] * x[i * d + k];
        const double norm = std::sqrt(s);
        if (norm > 1e-10) {
            const double inv = 1.0 / norm;
            for (int64_t k = 0; k < d; ++k) out[i * d + k] = x[i * d + k] * inv;
        } else {
            for (int64_t k = 0; k < d; ++k) out[i * d + k] = x[i * d + k];
        }
    }
}

// clusterWithCentroids (:39-92).  Returns the number of centroid rows written (k, or n when n <= k, or 0).
int32_t oracle_kmeans(const double *emb, int64_t n, int64_t d, int32_t num_clusters, int32_t max_iterations, uint64_t seed,
                      int32_t *labels, double *centroids, int32_t *iterations_out) {
    if (iterations_out) *iterations_out = 0;
    if (n <= 0) return 0;
    if (d <= 0) {
        for (int64_t i = 0; i < n; ++i) labels[i] = 0;
        return 0;
    }
    const int64_t k = std::min<int64_t>(num_clusters, n);
    if (k <= 0) {
        for (int64_t i = 0; i < n; ++i) labels[i] = 0;
        return 0;
    }
    if (n <= k) {                                            // :60-62: identity labels, centroids = raw embeddings
        for (int64_t i = 0; i < n; ++i) labels[i] = (int32_t)i;
        std::memcpy(centroids, emb, sizeof(double) * n * d);
        return (int32_t)n;
    }
    oracle_lcg rng{seed};
    std::vector<double> x((size_t)n * d);
    oracle_kmeans_normalize(emb, n, d, x.data());
    std::vector<int64_t> idx(n);
    for (int64_t i = 0; i < n; ++i) idx[i] = i;
    {   // indices.shuffle(using:)
        int64_t amount = n, cur = 0;
        while (amount > 1) {
            const int64_t r = (int64_t)rng.next_below((uint64_t)amount);
            amount -= 1;
            std::swap(idx[cur], idx[cur + r]);
            cur += 1;
        }
    }
    std::vector<double> c((size_t)k * d);
    for (int64_t j = 0; j < k; ++j) std::memcpy(&c[j * d], &x[idx[j] * d], sizeof(double) * d);
    std::vector<int32_t> assign(n, 0), fresh(n);
    std::vector<double> sums((size_t)k * d);
    std::vector<int64_t> counts(k);
    int it = 0;
    for (; it < max_iterations; ++it) {
        for (int64_t i = 0; i < n; ++i) {                    // assignToCentroids (:161-176): strict <, first minimum wins
            int32_t best = 0;
            double bd = std::numeric_limits<double>::max();
            for (int64_t j = 0; j < k; ++j) {
                const double dist = oracle_sqdist(&x[i * d], &c[j * d], d);
                if (dist < bd) {
                    bd = dist;
                    best = (int32_t)j;
                }
            }
            fresh[i] = best;
        }
        if (fresh == assign) break;
        assign = fresh;
        std::fill(sums.begin(), sums.end(), 0.0);            // updateCentroids (:187-210): sums in index order
        std::fill(counts.begin(), counts.end(), 0);
        for (int64_t i = 0; i < n; ++i) {
            const int32_t cl = assign[i];
            counts[cl] += 1;
            for (int64_t q = 0; q < d; ++q) sums[cl * d + q] += x[i * d + q];
        }
        for (int64_t j = 0; j < k; ++j) {
            if (counts[j] > 0) {
                const double inv = 1.0 / (double)counts[j];
                for (int64_t q = 0; q < d; ++q) c[j * d + q] = sums[j * d + q] * inv;
            } else {                                          // empty cluster: embeddings.randomElement(using:)
                const int64_t r = (int64_t)rng.next_below((uint64_t)n);
                std::memcpy(&c[j * d], &x[r * d], sizeof(double) * d);
            }
        }
    }
    if (iterations_out) *iterations_out = it;
    for (int64_t i = 0; i < n; ++i) labels[i] = assign[i];
    std::memcpy(centroids, c.data(), sizeof(double) * k * d);
    return (int32_t)k;
}

// clusterWithCentroidsNInit (:99-130): seeds base, base+1, ...; the lowest inertia wins, the first on ties
int32_t oracle_kmeans_ninit(const double *emb, int64_t n, int64_t d, int32_t num_clusters, int32_t max_iterations,
                            int32_t n_init, uint64_t base_seed, int32_t *labels, double *centroids, int32_t *best_init) {
    if (best_init) *best_init = 0;
    if (!(n > num_clusters && n_init > 1))
        return oracle_kmeans(emb, n, d, num_clusters, max_iterations, base_seed, labels, centroids, nullptr);
    std::vector<double> x((size_t)n * d);
    oracle_kmeans_normalize(emb, n, d, x.data());
    const int64_t kmax = std::max<int64_t>(1, std::min<int64_t>(num_clusters, n));
    std::vector<int32_t> lab(n);
    std::vector<double> cen((size_t)kmax * d);
    double best = std::numeric_limits<double>::max();
    int32_t best_k = -1;
    for (int32_t i = 0; i < n_init; ++i) {
        const int32_t k = oracle_kmeans(emb, n, d, num_clusters, max_iterations, base_seed + (uint64_t)i, lab.data(),
                                        cen.data(), nullptr);
        double inertia = 0.0;
        for (int64_t q = 0; q < n; ++q)
            if (lab[q] >= 0 && lab[q] < k) inertia += oracle_sqdist(&x[q * d], &cen[(int64_t)lab[q] * d], d);
        if (inertia < best) {
            best = inertia;
            best_k = k;
            std::memcpy(labels, lab.data(), sizeof(int32_t) * n);
            std::memcpy(centroids, cen.data(), sizeof(double) * (size_t)k * d);
            if (best_init) *best_init = i;
        }
    }
    if (best_k < 0) return oracle_kmeans(emb, n, d, num_clusters, max_iterations, base_seed, labels, centroids, nullptr);
    return best_k;
}

// SpeakerCountConstraints.resolve (:27-71); absent options (nil) are passed as INT64_MIN.  out = {min, max}.
void oracle_speaker_constraints(int64_t num_embeddings, int64_t num_speakers, int64_t min_speakers, int64_t max_speakers,
                                int64_t *out) {
    auto opt = [](int64_t v) { return v != INT64_MIN; };
    int64_t lo = opt(num_speakers) ? num_speakers : (opt(min_speakers) ? min_speakers : 1);
    lo = std::max<int64_t>(1, std::min(num_embeddings, lo));
    int64_t hi = opt(num_speakers) ? num_speakers : (opt(max_speakers) ? max_speakers : num_embeddings);
    hi = std::max<int64_t>(1, std::min(num_embeddings, hi));
    if (lo > hi) lo = hi;
    out[0] = lo;
    out[1] = hi;
}


// ---------------------------------------------------------------------------------------------------------------------
// Timeline reconstruction (SURVEY.md 8f rank 4, second half): OfflineReconstruction.buildSegments
//   Sources/FluidAudio/Diarizer/Offline/Utils/OfflineReconstruction.swift:24-253 (aggregation, per-frame speaker count,
//   ranking, segment accumulation), :399-425 appendSegment, :427-460 mergeSegments, :462-476 blendedQuality,
//   :478-493 sanitize, :359-397 excludeOverlaps, :495-505 chunkStartTime.
// Inputs are what the (not re-implemented) segmentation model produced: per chunk / frame / local-speaker weights.
// The optional zero-vote re-embed pass (:177-186) needs a span-embedding closure, i.e. model inference, and is disabled
// by default (OfflineDiarizerTypes.swift:279): not restated.
// "parity unpinned" in one respect: the reference closes and opens segments by iterating a Swift Dictionary / Set,
// whose order is randomised per process; only segments with EXACTLY equal start times can be reordered by that, and
// here they are taken in ascending cluster order (Swift's sort is stable, the later steps are order-preserving).
struct oracle_segment {
    int32_t cluster;
    float start, end, quality;
};
struct oracle_reconstruct_config {
    double frame_duration, window_duration, min_gap_duration, seg_min_duration_off, seg_min_duration_on, min_segment_duration;
    int32_t exclusive_segments;
};

static float oracle_blended_quality(const oracle_segment &l, const oracle_segment &r) {   // :462-476
    const double ld = (double)(l.end - l.start), rd = (double)(r.end - r.start), total = ld + rd;
    if (!(total > 0)) return std::min(std::max((l.quality + r.quality) / 2, 0.0f), 1.0f);
    const double weighted = (double)l.quality * ld + (double)r.quality * rd;
    return (float)std::min(std::max(weighted / total, 0.0), 1.0);
}

int32_t oracle_build_segments(const float *weights, int32_t num_chunks, int32_t num_frames, int32_t num_speakers,
                              const double *chunk_offsets, int32_t offsets_count, const int32_t *hard_clusters,
                              int32_t hard_rows, int32_t centroid_count, const oracle_reconstruct_config *cfg,
                              oracle_segment *out, int32_t cap) {
    if (num_chunks <= 0 || num_frames <= 0) return 0;
    const double dur = cfg->frame_duration;
    if (!(dur > 0)) return 0;
    const int K = std::max(centroid_count, 1);
    const double gap_threshold = std::max(cfg->min_gap_duration, cfg->seg_min_duration_off);
    auto chunk_start = [&](int c) { return c < offsets_count ? chunk_offsets[c] : (double)c * cfg->window_duration; };
    double max_time = 0.0;
    for (int c = 0; c < num_chunks; ++c) max_time = std::max(max_time, chunk_start(c) + (double)num_frames * dur);
    const int total = std::max(1, (int)std::ceil(max_time / dur));
    std::vector<std::vector<double>> sums(total, std::vector<double>(K, 0.0)), counts(total, std::vector<double>(K, 0.0));
    std::vector<double> exp_sum(total, 0.0), exp_w(total, 0.0);
    for (int c = 0; c < num_chunks; ++c) {
        const double off = chunk_start(c);
        for (int f = 0; f < num_frames; ++f) {
            const double fs = off + (double)f * dur;
            int g = (int)std::round(fs / dur);                       // .rounded(): to nearest, ties away from zero
            g = std::min(std::max(g, 0), total - 1);
            const float *w = weights + ((size_t)c * num_frames + f) * num_speakers;
            std::vector<double> act(K, 0.0);
            for (int s = 0; s < num_speakers; ++s) {
                const int cl = c < hard_rows ? hard_clusters[(size_t)c * num_speakers + s] : -2;
                if (cl < 0 || cl >= K) continue;
                if ((double)w[s] > act[cl]) act[cl] = (double)w[s];
            }
            double expected = 0.0;
            for (int s = 0; s < num_speakers; ++s) expected += (double)w[s];
            exp_sum[g] += expected;
            exp_w[g] += 1;
            for (int k = 0; k < K; ++k)
                if (act[k] > 0) {
                    sums[g][k] += act[k];
                    counts[g][k] += 1;
                }
        }
    }
    std::vector<std::vector<double>> avg(total, std::vector<double>(K, 0.0));
    for (int g = 0; g < total; ++g)
        for (int k = 0; k < K; ++k) avg[g][k] = counts[g][k] == 0 ? 0.0 : sums[g][k] / counts[g][k];
    const int max_allowed = std::min(K, num_speakers);
    std::vector<std::vector<int>> per_frame(total);
    for (int g = 0; g < total; ++g) {
        if (!(exp_w[g] > 0)) continue;
        int required = (int)std::nearbyint(exp_sum[g] / exp_w[g]);   // .toNearestOrEven (default FE_TONEAREST)
        required = std::min(std::max(required, 0), max_allowed);
        if (required <= 0) continue;
        std::vector<int> order(K);
        for (int k = 0; k < K; ++k) order[k] = k;
        std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return sums[g][a] > sums[g][b]; });
        per_frame[g].assign(order.begin(), order.begin() + required);
    }
    struct Acc {
        bool on = false;
        double start = 0, end = 0, score = 0;
        int frames = 0;
    };
    std::vector<Acc> active(K);
    std::vector<oracle_segment> raw;
    auto append = [&](int k, const Acc &a, double end_time) {        // appendSegment (:399-425)
        if (!(end_time > a.start)) return;
        const double mean = a.frames > 0 ? a.score / (double)a.frames : a.score;
        raw.push_back({k, (float)a.start, (float)end_time, (float)std::min(std::max(mean, 0.0), 1.0)});
    };
    for (int g = 0; g < total; ++g) {
        const double fs = (double)g * dur, fe = fs + dur;
        std::vector<char> now(K, 0);
        for (int k : per_frame[g]) now[k] = 1;
        for (int k = 0; k < K; ++k)
            if (active[k].on && !now[k]) {
                append(k, active[k], fs);
                active[k] = Acc{};
            }
        for (int k = 0; k < K; ++k) {
            if (!now[k]) continue;
            if (active[k].on) {
                active[k].end = fe;
                active[k].score += avg[g][k];
                active[k].frames += 1;
            } else {
                active[k].on = true;
                active[k].start = fs;
                active[k].end = fe;
                active[k].score = avg[g][k];
                active[k].frames = 1;
            }
        }
    }
    for (int k = 0; k < K; ++k)
        if (active[k].on) append(k, active[k], active[k].end);
    // mergeSegments (:427-460)
    std::vector<oracle_segment> merged;
    if (!raw.empty()) {
        std::stable_sort(raw.begin(), raw.end(), [](const oracle_segment &a, const oracle_segment &b) { return a.start < b.start; });
        oracle_segment cur = raw[0];
        for (size_t i = 1; i < raw.size(); ++i) {
            const oracle_segment &sg = raw[i];
            if (sg.cluster == cur.cluster && (double)sg.start - (double)cur.end <= gap_threshold) {
                const float q = oracle_blended_quality(cur, sg);
                cur.end = std::max(cur.end, sg.end);
                cur.quality = q;
                continue;
            }
            merged.push_back(cur);
            cur = sg;
        }
        merged.push_back(cur);
    }
    // sanitize (:478-493)
    std::stable_sort(merged.begin(), merged.end(), [](const oracle_segment &a, const oracle_segment &b) { return a.start < b.start; });
    const float min_dur = std::max((float)cfg->min_segment_duration, (float)cfg->seg_min_duration_on);
    std::vector<oracle_segment> kept;
    for (const auto &sg : merged)
        if (sg.end - sg.start >= min_dur) kept.push_back(sg);
    std::vector<oracle_segment> result;
    if (cfg->exclusive_segments) {                                    // excludeOverlaps (:359-397)
        for (const auto &sg : kept) {
            float st = sg.start;
            const float en = sg.end;
            if (!result.empty() && st < result.back().end) st = result.back().end;
            if (st >= en) continue;
            const float d = en - st;
            if (d < (float)cfg->min_segment_duration) continue;
            const float orig = sg.end - sg.start;
            const float scale = orig > 0 ? d / orig : 1.0f;
            result.push_back({sg.cluster, st, en, std::max(0.0f, std::min(1.0f, sg.quality * scale))});
        }
    } else {
        result = kept;
    }
    const int32_t n = (int32_t)result.size();
    for (int32_t i = 0; i < n && i < cap; ++i) out[i] = result[i];
    return n;
}


// OfflineReconstruction.buildSpeakerDatabase (OfflineReconstruction.swift:296-357): per speaker the float32 mean of its
// segments' embeddings; a segment's embedding is its cluster's centroid narrowed to Float (appendSegment :409-414, zeros
// when the cluster has no centroid).  database: [K x dim], rows of speakers without segments stay zero; counts: [K].
void oracle_build_speaker_database(const int32_t *seg_cluster, int32_t seg_count, const double *centroids, int32_t K,
                                   int32_t dim, float *database, int32_t *counts) {
    for (int32_t k = 0; k < K; ++k) counts[k] = 0;
    for (int64_t i = 0; i < (int64_t)K * dim; ++i) database[i] = 0.0f;
    for (int32_t s = 0; s < seg_count; ++s) {
        const int32_t k = seg_cluster[s];
        if (k < 0 || k >= K) continue;
        for (int32_t q = 0; q < dim; ++q) {
            const float e = (float)centroids[(int64_t)k * dim + q];
            database[(int64_t)k * dim + q] = counts[k] == 0 ? e : database[(int64_t)k * dim + q] + e;   // first: copy (:330)
        }
        counts[k] += 1;
    }
    for (int32_t k = 0; k < K; ++k) {
        if (counts[k] <= 0) continue;
        const float scale = 1.0f / (float)counts[k];
        for (int32_t q = 0; q < dim; ++q) database[(int64_t)k * dim + q] *= scale;
    }
}

} // extern "C"
