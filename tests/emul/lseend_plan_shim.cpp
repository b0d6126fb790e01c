// C entry points over the LS-EEND streams' planning arithmetic (fluidaudio_b200/csrc/lseend/lseend_plan.h, compiled with this
// file by g++), for tests/test_lseend_streams.py: the derived sizes and one push's step, as every push plans them.
#include "lseend_plan.h"

#include <cstdarg>
#include <cstdio>

namespace fa {
static char g_error[512] = "";
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}
const char *last_error() { return g_error; }
} // namespace fa

using namespace fa::lseend;

extern "C" {

const char *lp_last_error() { return fa::last_error(); }

// cfg: {sample_rate, n_mels, hop, win, context, subsampling, chunk, conv_delay, precision}; sizes: the 10 of Sizes
int lp_resolve(const int *cfg, int *sizes) {
    const Config c{cfg[0], cfg[1], cfg[2], cfg[3], cfg[4], cfg[5], cfg[6], cfg[7], cfg[8]};
    Sizes s;
    const int st = resolve(c, s);
    if (st == FA_OK) {
        const int v[10] = {s.n_fft,         s.mel_frames,  s.chunk_mels,    s.mel_context, s.chunk_samples,
                           s.audio_left,    s.audio_context, s.flush_samples, s.mask_length, s.audio_capacity};
        for (int i = 0; i < 10; ++i) sizes[i] = v[i];
    }
    return st;
}

// lengths in/out: {audio, mel, cmn_count, mask_end} (a fresh session when fresh != 0); out: {zeros, unread, consumed,
// frames, chunks}.  Also the mask windows and warm-up counts of the push's chunks: masks [chunks x chunk], warmup [chunks].
int lp_step(const int *cfg, int fresh_session, long long *lengths, long long n, int drain, long long *out, float *masks,
            int *warmup) {
    const Config c{cfg[0], cfg[1], cfg[2], cfg[3], cfg[4], cfg[5], cfg[6], cfg[7], cfg[8]};
    Sizes s;
    const int st = resolve(c, s);
    if (st != FA_OK) return st;
    const Lengths m = fresh_session ? fresh(c, s) : Lengths{lengths[0], lengths[1], lengths[2], (int)lengths[3]};
    const Step t = plan_push(c, s, m, n, drain != 0);
    const long long v[5] = {t.zeros, t.unread, t.consumed, t.frames, t.chunks};
    for (int i = 0; i < 5; ++i) out[i] = v[i];
    for (long long j = 0; j < t.chunks; ++j) {
        const int end = (int)std::min<long long>(m.mask_end + (j + 1) * c.chunk_size, s.mask_length);
        for (int k = 0; k < c.chunk_size; ++k) masks[j * c.chunk_size + k] = mask_value(end, c.chunk_size, c.conv_delay, k);
        warmup[j] = warmup_frames(end, c.chunk_size, s.mask_length);
    }
    lengths[0] = t.next.audio;
    lengths[1] = t.next.mel;
    lengths[2] = t.next.cmn_count;
    lengths[3] = t.next.mask_end;
    return FA_OK;
}

} // extern "C"
