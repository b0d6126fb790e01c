// Host run of Sortformer's per-element arithmetic (fluidaudio_b200/csrc/sortformer_core.cuh; CPU test-suite only): the
// functions sortformer_update_kernel calls, driven element by element in the kernel's phases.
//   sortformer_emul_compress(preds [L x 4], L, spkcache_len, sil, thr, boost_latest, strong_k, weak_k, min_pos,
//                            scores, disabled, strong, weak [L x 4], slot [spkcache_len])
//       slot[r] = the kept frame of output row r, or -1 for a disabled row (silence mean, zero predictions)
//   sortformer_emul_silence(embs [n x 512], preds [n x 4], n, silence_threshold, mean [512] in/out, count in/out)
#include "../../fluidaudio_b200/csrc/sortformer_core.cuh"

#include <vector>

using namespace fa::sortformer;

static void boost_phase(std::vector<float> &s, int L, int k, float scale) {
    if (k <= 0) return;
    std::vector<int> flag(s.size(), 0);
    for (int i = 0; i < L * kSpeakers; ++i) {
        const float v = s[i];
        const int spk = i & 3;
        flag[i] = v != -INFINITY && rank_until([&](int g) { return s[g * kSpeakers + spk]; }, L, v, i >> 2, k, true) < k;
    }
    for (int i = 0; i < L * kSpeakers; ++i)
        if (flag[i]) s[i] = boost(s[i], scale);
}

extern "C" void sortformer_emul_compress(const float *preds, int L, int K, int sil, float thr, float boost_latest,
                                         int strong_k, int weak_k, int min_pos, float *scores_out, float *disabled_out,
                                         float *strong_out, float *weak_out, int *slot) {
    std::vector<float> s(L * kSpeakers);
    for (int f = 0; f < L; ++f) frame_scores(preds + f * kSpeakers, thr, s.data() + f * kSpeakers);
    for (int i = 0; i < L * kSpeakers; ++i) scores_out[i] = s[i];
    int pos[kSpeakers] = {0, 0, 0, 0};
    for (int i = 0; i < L * kSpeakers; ++i) pos[i & 3] += positive_score(preds[i], s[i]) ? 1 : 0;
    for (int i = 0; i < L * kSpeakers; ++i)
        s[i] = disable_and_boost(preds[i], s[i], pos[i & 3], min_pos, (i >> 2) >= K, boost_latest);
    for (int i = 0; i < L * kSpeakers; ++i) disabled_out[i] = s[i];
    boost_phase(s, L, strong_k, 2.0f);
    for (int i = 0; i < L * kSpeakers; ++i) strong_out[i] = s[i];
    boost_phase(s, L, weak_k, 1.0f);
    for (int i = 0; i < L * kSpeakers; ++i) weak_out[i] = s[i];
    const int F = L + sil, N = F * kSpeakers;
    std::vector<float> perm(N);
    for (int p = 0; p < N; ++p) {
        const int spk = p / F, f = p - spk * F;
        perm[p] = f < L ? s[f * kSpeakers + spk] : INFINITY;
    }
    for (int r = 0; r < K; ++r) slot[r] = -1;
    int at = 0;
    for (int p = 0; p < N; ++p) {
        const float v = perm[p];
        if (rank_until([&](int q) { return perm[q]; }, N, v, p, K, false) < K && kept_index(v, p) != kMaxIndex) {
            const int f = p % F;
            if (at < K) slot[at] = f < L ? f : -1;
            ++at;
        }
    }
}

extern "C" void sortformer_emul_silence(const float *embs, const float *preds, int n, float threshold, float *mean,
                                        long long *count) {
    for (int j = 0; j < n; ++j) {
        if (!(prob_sum(preds + j * kSpeakers) < threshold)) continue;
        const float nf = (float)*count;
        for (int d = 0; d < kDims; ++d) mean[d] = mean_step(mean[d], embs[(size_t)j * kDims + d], nf);
        ++*count;
    }
}
