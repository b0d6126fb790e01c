// Host run of offline Sortformer window arithmetic (fluidaudio_b200/csrc/offline_sortformer/offline_sortformer_core.cuh;
// CPU test-suite only), in the kernels' own formulation: the closed-form window count, the packed permutation order,
// the correlation chains, the scores and the choice, and one file's stitching with coverage as a prefix.
#include "../../fluidaudio_b200/csrc/offline_sortformer/offline_sortformer_core.cuh"

#include <cfloat>
#include <cstdint>

using namespace fa::offline_sortformer;

namespace {

// the stitcher's choice over the staged overlap rows, sequentially: the first score strictly above the best so far
int choose(const float *global, const float *window, int ov) {
    float c[kSpeakers][kSpeakers];
    for (int g = 0; g < kSpeakers; ++g)
        for (int w = 0; w < kSpeakers; ++w) c[g][w] = correlation(global, window, ov, g, w);
    int best = 0;
    float best_score = -FLT_MAX;
    for (int p = 0; p < kPerms; ++p) {
        const float s = score(c[0][perm_at(p, 0)], c[1][perm_at(p, 1)], c[2][perm_at(p, 2)], c[3][perm_at(p, 3)]);
        if (s > best_score) best_score = s, best = p;
    }
    return best;
}

void invert(int p, int32_t *mapping) {
    for (int g = 0; g < kSpeakers; ++g) mapping[perm_at(p, g)] = g;
}

} // namespace

extern "C" {

int osf_emul_clamp(int overlap) { return clamp_overlap(overlap); }

void osf_emul_plan(int overlap, int64_t mel_frames, int64_t *windows, int64_t *rows) {
    *windows = window_count(mel_frames, clamp_overlap(overlap));
    *rows = total_out(mel_frames);
}

int osf_emul_perm(int p, int g) { return perm_at(p, g); }

// mapping [4] over `frames` overlap rows [frames x 4] of the timeline and the window
void osf_emul_alignment(const float *global, const float *window, int frames, int32_t *mapping) {
    invert(frames > 0 ? choose(global, window, frames) : 0, mapping);
}

// one file's stitching: preds [windows x 384 x 4] -> out [totalOut x 4], mappings [windows x 4]
void osf_emul_stitch(int overlap, int64_t mel_frames, const float *preds, float *out, int32_t *mappings) {
    overlap = clamp_overlap(overlap);
    const long long total = total_out(mel_frames), windows = window_count(mel_frames, overlap);
    long long covered = 0;
    float staged[2][(kWindowOut - 1) * kSpeakers];
    for (long long k = 0; k < windows; ++k) {
        const Window win = window_at(mel_frames, overlap, k);
        const long long g_start = win.mel_start / kSubsampling;
        const float *P = preds + k * kWindowOut * kSpeakers;
        const int ov = k > 0 && overlap > 0 ? overlap_frames(overlap, win.valid_out, total, g_start) : 0;
        int best = 0;
        if (ov > 0) {
            for (int e = 0; e < ov * kSpeakers; ++e) {
                staged[0][e] = out[g_start * kSpeakers + e];
                staged[1][e] = P[e];
            }
            best = choose(staged[0], staged[1], ov);
        }
        int32_t *m = mappings + k * kSpeakers;
        invert(best, m);
        for (int j = 0; j < win.valid_out; ++j) {
            const long long gf = g_start + j;
            if (gf >= total) break;
            for (int w = 0; w < kSpeakers; ++w) {
                float *dst = out + gf * kSpeakers + m[w];
                *dst = gf < covered ? average(*dst, P[j * kSpeakers + w]) : P[j * kSpeakers + w];
            }
        }
        const long long end = g_start + win.valid_out < total ? g_start + win.valid_out : total;
        covered = end > covered ? end : covered;
    }
}

} // extern "C"
