// Host run of voice activity detection's arithmetic (fluidaudio_b200/csrc/vad/vad_core.cuh; CPU test-suite only), in
// the kernels' own formulation: the chunk staging per sample, the streaming step, speech segmentation with its three
// running candidates and the one-range padding lag, and the FSMN decision with its bit-mask window.
//   vad_emul_chunk_sample(x, n, j)                       sample j of the processed chunk
//   vad_emul_stream_step(state, p, n, resolved, sample)  state = {processed, triggered, temp_end}; the event kind
//   vad_emul_segment(p, P, L, resolved, out)             pairs into out (at most P); their count
//   vad_emul_fsmn(sil, T, out)                           pairs into out (at most (T + 1) / 2); their count
#include "../../fluidaudio_b200/csrc/vad/vad_core.cuh"

#include <cstdint>

using namespace fa::vad;

namespace {

struct CResolved {   // fa_vad_resolved's layout
    float threshold, negative, split;
    int32_t use_max;
    int64_t min_speech, min_silence, max_speech, pad, min_silence_at_max;
};

Resolved of(const CResolved *c) {
    return Resolved{c->threshold,    c->negative,    c->split, c->use_max,          c->min_speech,
                    c->min_silence, c->max_speech, c->pad,   c->min_silence_at_max};
}

} // namespace

extern "C" {

float vad_emul_chunk_sample(const float *x, int64_t n, int j) { return chunk_sample(x, n, j); }

int vad_emul_stream_step(int64_t *state, float p, int64_t n, const CResolved *r, int64_t *sample) {
    StreamState s{state[0], state[2], state[1]};
    long long e;
    const int kind = stream_step(s, p, n, of(r), &e);
    state[0] = s.processed;
    state[1] = s.triggered;
    state[2] = s.temp_end;
    *sample = e;
    return kind;
}

int64_t vad_emul_segment(const float *p, int64_t P, int64_t L, const CResolved *r, int64_t *out) {
    return segment_clip(p, P, L, of(r), reinterpret_cast<long long *>(out));
}

int64_t vad_emul_fsmn(const float *sil, int64_t T, int64_t *out) {
    return fsmn_clip(sil, T, reinterpret_cast<long long *>(out));
}

} // extern "C"
