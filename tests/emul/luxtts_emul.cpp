// Host run of LuxTTS synthesis arithmetic (fluidaudio_b200/csrc/luxtts/luxtts_core.cuh; CPU test-suite only), in the
// kernels' own formulation: counter-based SplitMix64 draws, Box-Muller on the host libm, the float32 anchor-Euler
// update, the RMS tree and the plan.
#include "../../fluidaudio_b200/csrc/luxtts/luxtts_core.cuh"

#include <cstdint>

using namespace fa::luxtts;

extern "C" {

double luxtts_emul_uniform(uint64_t seed, uint64_t k) { return uniform_at(seed_state(seed), k); }

void luxtts_emul_noise(uint64_t seed, int64_t count, float *out) {
    for (int64_t j = 0; j < count; ++j) out[j] = gaussian_at(seed_state(seed), (uint64_t)j);
}

void luxtts_emul_step(float *x, const float *v, int64_t n, int step) {
    const float tc = (float)time_step(step), tn = (float)time_step(step + 1);
    for (int64_t i = 0; i < n; ++i) x[i] = anchor_euler(x[i], v[i], tc, tn, step == kSteps - 1);
}

float luxtts_emul_rms(const float *x, int64_t n) { return rms_tree(x, n); }

double luxtts_emul_time_step(int i) { return time_step(i); }

int luxtts_emul_plan(int64_t samples, int32_t pt, int32_t tt, float speed, int32_t *out) {
    const Plan p = plan_request(samples, pt, tt, speed);
    const int32_t v[6] = {p.prompt_samples, p.prompt_frames, p.token_count, p.features_length, p.gen_frames, p.bucket};
    for (int i = 0; i < 6; ++i) out[i] = v[i];
    return p.reason;
}

float luxtts_emul_clip(float x) { return clip_unit(x); }

} // extern "C"
