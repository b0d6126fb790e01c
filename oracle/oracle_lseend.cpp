// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the shipped product path.
//
// Sequential CPU restatement of LSEENDFeatureProvider (Sources/FluidAudio/Diarizer/LS-EEND/LSEENDPreprocessor.swift),
// one provider per object, line by line: init (:46-114), enqueueAudio (:123-141), drainRightContextWithSilence
// (:158-180), emitNextChunk (:185-202), takeSnapshot / rollback / reset (:206-245), processAudioQueue (:249-279) and
// StreamingChunkQueue (:284-384), with the metadata's derived sizes (LSEENDTypes.swift:53-57).  The log-mel is the main
// oracle's AudioMelSpectrogram restatement (oracle_mel.cpp, precision 0) and the scaling and running mean its LS-EEND
// restatement (oracle_adapters.cpp); both are compiled into this library with the main oracle's pinned flags.

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

extern "C" {
struct oracle_mel_config {
    int32_t sample_rate, n_mels, n_fft, hop_length, win_length;
    float preemph;
    int32_t pad_to;
    float log_floor;
    int32_t log_floor_mode, window_periodic, precision;
};
int64_t oracle_mel_compute_flat_transposed(const oracle_mel_config *c, const float *audio, int64_t n, float last_sample,
                                           int32_t padding_mode, int64_t expected, float *out, int64_t out_len,
                                           int64_t *mel_length, int64_t *num_frames);
void oracle_lseend_scale_cmn(float *x, int64_t frames, int32_t n_mels, float *cmn_mean, int64_t *cmn_count);
}

namespace {

// StreamingChunkQueue (:284-384).  The reference trims its buffer lazily to bound memory; which elements are unread
// does not depend on when it trims, so this one keeps everything and moves the head.
struct ChunkQueue {
    int64_t stride, context, chunk, padded, left;
    int64_t head = 0;
    std::vector<float> buffer;

    ChunkQueue(int64_t chunk_length, int64_t left_context, int64_t right_context, int64_t stride_)
        : stride(stride_), context((left_context + right_context) * stride_), chunk(chunk_length * stride_),
          padded(chunk_length * stride_ + (left_context + right_context) * stride_), left(left_context * stride_) {
        buffer.assign(left, 0.0f);
    }
    int64_t unread() const { return (int64_t)buffer.size() - head; }
    int64_t ready() const { return std::max<int64_t>(0, (unread() - context) / chunk); }
    bool has_chunk() const { return unread() >= padded; }
    void append(const float *x, int64_t n) { buffer.insert(buffer.end(), x, x + n); }
    void append_zeros(int64_t n) { buffer.insert(buffer.end(), (size_t)n, 0.0f); }
    // popNextChunk: [head, head + padded), head += chunk
    bool pop_next(std::vector<float> &out) {
        if (!has_chunk()) return false;
        out.assign(buffer.begin() + head, buffer.begin() + head + padded);
        head += chunk;
        return true;
    }
    // popAllChunks: [head, newHead + context), head = newHead
    bool pop_all(std::vector<float> &out) {
        if (!has_chunk()) return false;
        const int64_t new_head = head + ((int64_t)buffer.size() - head - context) / chunk * chunk;
        out.assign(buffer.begin() + head, buffer.begin() + new_head + context);
        head = new_head;
        return true;
    }
    void reset() {
        head = 0;
        buffer.assign(left, 0.0f);
    }
};

struct Provider {
    oracle_mel_config mel;
    int32_t n_mels, chunk_frames, flush;
    std::vector<float> decoder_mask;
    ChunkQueue mel_q, audio_q;
    std::vector<float> cmn_mean;
    int64_t cmn_count = 0;
    int32_t mask_end = 0;
    struct Snapshot {
        ChunkQueue mel_q, audio_q;
        std::vector<float> cmn_mean;
        int64_t cmn_count;
        int32_t mask_end;
    };
    std::vector<Snapshot> snapshot;   // zero or one

    // :46-114; ints = {sampleRate, nMels, hopLength, winLength, contextSize, subsampling, chunkSize, convDelay}
    static int32_t next_pow2(int32_t w) {
        int32_t n = 1;
        while (n < w) n <<= 1;
        return n;
    }
    explicit Provider(const int32_t *v)
        : n_mels(v[1]), chunk_frames(v[6]),
          flush((v[4] + v[7] * v[5]) * v[2] + next_pow2(v[3]) / 2),
          mel_q(v[5] * v[6], v[4], v[4] + 1 - v[5], v[1]),
          audio_q((int64_t)v[2] * v[5] * v[6], next_pow2(v[3]) / 2, next_pow2(v[3]) / 2 - v[2], 1),
          cmn_mean(v[1], 0.0f) {
        mel = oracle_mel_config{v[0], v[1], next_pow2(v[3]), v[2], v[3], 0.0f, 0, 1e-10f, 1, 1, 0};
        decoder_mask.assign(v[7] + v[6], 1.0f);
        std::fill(decoder_mask.begin(), decoder_mask.begin() + v[7], 0.0f);
    }

    // :249-279
    void process_audio_queue() {
        std::vector<float> chunk;
        if (!audio_q.pop_all(chunk)) return;
        int64_t ml = 0, nf = 0;
        const int64_t need = oracle_mel_compute_flat_transposed(&mel, chunk.data(), (int64_t)chunk.size(), 0.0f, 1, -1,
                                                                nullptr, 0, &ml, &nf);
        std::vector<float> feats(need);
        oracle_mel_compute_flat_transposed(&mel, chunk.data(), (int64_t)chunk.size(), 0.0f, 1, -1, feats.data(), need, &ml,
                                           &nf);
        oracle_lseend_scale_cmn(feats.data(), ml, n_mels, cmn_mean.data(), &cmn_count);
        mel_q.append(feats.data(), ml * n_mels);
    }
    // :123-141 (eager)
    void enqueue(const float *x, int64_t n) {
        audio_q.append(x, n);
        process_audio_queue();
    }
    // :158-180 (flush: true)
    void drain() {
        audio_q.append_zeros(flush);
        const int64_t over = std::max<int64_t>(0, audio_q.unread() - audio_q.context);
        const int64_t shortfall = (audio_q.chunk - over % audio_q.chunk) % audio_q.chunk;
        if (shortfall > 0) audio_q.append_zeros(shortfall);
        process_audio_queue();
    }
    // :185-202
    bool emit(float *features, float *mask, int32_t *warmup) {
        process_audio_queue();
        std::vector<float> raw;
        if (!mel_q.pop_next(raw)) return false;
        mask_end = std::min<int32_t>(mask_end + chunk_frames, (int32_t)decoder_mask.size());
        std::memcpy(features, raw.data(), raw.size() * sizeof(float));
        std::memcpy(mask, decoder_mask.data() + mask_end - chunk_frames, (size_t)chunk_frames * sizeof(float));
        *warmup = std::min<int32_t>((int32_t)decoder_mask.size() - mask_end, chunk_frames);
        return true;
    }
    void take_snapshot() { snapshot.assign(1, Snapshot{mel_q, audio_q, cmn_mean, cmn_count, mask_end}); }
    void rollback() {
        const Snapshot &s = snapshot.at(0);
        mel_q = s.mel_q;
        audio_q = s.audio_q;
        cmn_mean = s.cmn_mean;
        cmn_count = s.cmn_count;
        mask_end = s.mask_end;
    }
    void reset() {
        std::fill(cmn_mean.begin(), cmn_mean.end(), 0.0f);
        cmn_count = 0;
        mask_end = 0;
        audio_q.reset();
        mel_q.reset();
    }
};

} // namespace

extern "C" {

void *oracle_lseend_create(const int32_t *ints) { return new Provider(ints); }
void oracle_lseend_destroy(void *p) { delete static_cast<Provider *>(p); }
void oracle_lseend_enqueue(void *p, const float *x, int64_t n) { static_cast<Provider *>(p)->enqueue(x, n); }
void oracle_lseend_drain(void *p) { static_cast<Provider *>(p)->drain(); }
int64_t oracle_lseend_ready(const void *p) { return static_cast<const Provider *>(p)->mel_q.ready(); }
int32_t oracle_lseend_emit(void *p, float *features, float *mask, int32_t *warmup) {
    return static_cast<Provider *>(p)->emit(features, mask, warmup) ? 1 : 0;
}
void oracle_lseend_snapshot(void *p) { static_cast<Provider *>(p)->take_snapshot(); }
void oracle_lseend_rollback(void *p) { static_cast<Provider *>(p)->rollback(); }
void oracle_lseend_reset(void *p) { static_cast<Provider *>(p)->reset(); }
// lengths: {unread audio samples, unread mel rows, cmnCount, decoderMaskEnd}
void oracle_lseend_lengths(const void *p, int64_t *v) {
    const Provider *q = static_cast<const Provider *>(p);
    v[0] = q->audio_q.unread();
    v[1] = q->mel_q.unread() / q->n_mels;
    v[2] = q->cmn_count;
    v[3] = q->mask_end;
}
// audio [unread samples], mel [unread rows x nMels], cmn_mean [nMels]
void oracle_lseend_state(const void *p, float *audio, float *mel, float *cmn_mean) {
    const Provider *q = static_cast<const Provider *>(p);
    std::copy(q->audio_q.buffer.begin() + q->audio_q.head, q->audio_q.buffer.end(), audio);
    std::copy(q->mel_q.buffer.begin() + q->mel_q.head, q->mel_q.buffer.end(), mel);
    std::copy(q->cmn_mean.begin(), q->cmn_mean.end(), cmn_mean);
}

} // extern "C"
