// Host run of the prepare stage's per-element arithmetic (fluidaudio_b200/csrc/prepare_core.cuh; CPU test-suite only):
// the functions the kernels call, driven frame by frame and speaker by speaker as the kernels drive them.
//   prepare_emul_decode(logits, frames, classes, onset, log_probs, weights[frames x 3], histogram[8]) -> speech frames
//   prepare_emul_resample(rows, row_count, in_len, out_len, out)
//   prepare_emul_interp(in_len, out_len, left, right, w_left, w_right)
//   prepare_emul_speaker(w[frames x speakers], frames, speakers, s, exclude, min_frames, weight_frames,
//                        mask[frames], resampled[weight_frames], out[5] = emit, fallback, first, last, clean;
//                        sums[3] = maskSum, energy, baseSum)   embedding_mask_kernel + embedding_pack_kernel for one speaker
//   prepare_emul_cosine(a, b, n)      mask_reuse_kernel's similarity (lane-strided dot products, xor butterfly)
//   prepare_emul_time(offset, frame, frame_duration)
#include "../../fluidaudio_b200/csrc/prepare_core.cuh"

#include <climits>
#include <vector>

using namespace fa::prepare;

extern "C" long long prepare_emul_decode(const float *logits, long long frames, int classes, float onset, float *log_probs,
                                         float *weights, long long *histogram) {
    long long speech = 0;
    for (int k = 0; k < kPowersetClasses; ++k) histogram[k] = 0;
    for (long long f = 0; f < frames; ++f) {
        std::vector<float> row(logits + f * classes, logits + (f + 1) * classes);
        const FrameDecision d = decode_frame(row.data(), classes, onset, row.data());   // in place, as the kernel does
        for (int c = 0; c < classes; ++c) log_probs[f * classes + c] = row[c];
        if (d.best < kPowersetClasses) histogram[d.best] += 1;
        speech += d.speech;
        const unsigned who = powerset_speakers(d.best < kPowersetClasses - 1 ? d.best : kPowersetClasses - 1);
        for (int s = 0; s < kDecodeSpeakers; ++s) weights[f * kDecodeSpeakers + s] = (who >> s) & 1u ? 1.0f : 0.0f;
    }
    return speech;
}

extern "C" void prepare_emul_resample(const float *rows, long long row_count, int in_len, int out_len, float *out) {
    for (long long r = 0; r < row_count; ++r)
        for (int i = 0; i < out_len; ++i) out[r * out_len + i] = resample_at(rows + r * in_len, in_len, out_len, i);
}

extern "C" void prepare_emul_interp(int in_len, int out_len, int *left, int *right, float *w_left, float *w_right) {
    for (int i = 0; i < out_len; ++i) {
        const Interp k = interp_coefficients(i, in_len, out_len);
        left[i] = k.left;
        right[i] = k.right;
        w_left[i] = k.w_left;
        w_right[i] = k.w_right;
    }
}

extern "C" void prepare_emul_speaker(const float *w, int frames, int speakers, int s, int exclude, int min_frames,
                                     int weight_frames, float *mask, float *resampled, int *out, float *sums) {
    std::vector<unsigned char> overlap(frames, 0);
    for (int f = 0; f < frames; ++f) {
        int active = 0;
        for (int k = 0; k < speakers; ++k) active += w[f * speakers + k] > kActiveThreshold ? 1 : 0;
        overlap[f] = exclude && active > 1;
    }
    auto base = [&](int f) { return w[f * speakers + s]; };
    auto clean = [&](int f) { return overlap[f] ? 0.0f : w[f * speakers + s]; };
    const float base_sum = ordered_sum(base, frames), clean_sum = ordered_sum(clean, frames);
    const MaskDecision d = mask_decide(base_sum, clean_sum, frames, min_frames);
    out[0] = 0;
    out[1] = d.fallback;
    out[4] = d.use_clean;
    sums[0] = d.mask_sum;
    sums[1] = 0.0f;
    sums[2] = base_sum;
    if (!d.candidate) return;
    int first = INT_MAX, last = -1;
    for (int f = 0; f < frames; ++f) {
        mask[f] = d.use_clean ? clean(f) : base(f);
        if (mask[f] > kActiveThreshold) {
            first = first < f ? first : f;
            last = f;
        }
    }
    for (int j = 0; j < weight_frames; ++j) resampled[j] = resample_at(mask, frames, weight_frames, j);
    sums[1] = ordered_sum([&](int j) { return resampled[j]; }, weight_frames);
    out[0] = sums[1] <= 0.0f ? 0 : 1;
    out[2] = first == INT_MAX ? 0 : first;
    out[3] = last < 0 ? out[2] : last;
}

extern "C" float prepare_emul_cosine(const float *a, const float *b, int n) {
    float dot[32], na[32], nb[32];
    for (int lane = 0; lane < 32; ++lane) {
        dot[lane] = na[lane] = nb[lane] = 0.0f;
        for (int f = lane; f < n; f += 32) {
            dot[lane] = f_add(dot[lane], f_mul(a[f], b[f]));
            na[lane] = f_add(na[lane], f_mul(a[f], a[f]));
            nb[lane] = f_add(nb[lane], f_mul(b[f], b[f]));
        }
    }
    for (int m = 16; m > 0; m >>= 1)
        for (int lane = 0; lane < m; ++lane) {   // lane 0's value after the butterfly
            dot[lane] = f_add(dot[lane], dot[lane + m]);
            na[lane] = f_add(na[lane], na[lane + m]);
            nb[lane] = f_add(nb[lane], nb[lane + m]);
        }
    return mask_cosine(dot[0], na[0], nb[0]);
}

extern "C" double prepare_emul_time(double offset, int frame, double frame_duration) {
    return frame_time(offset, frame, frame_duration);
}
