// Host side of CTC keyword spotting (ctc_kernels.cu), behind the C ABI of ctc_abi.cu.  Arguments reach these functions
// already checked; each returns an FA_* status.
#pragma once

#include "../../../include/fluidaudio_b200_ctc.h"
#include "../call_context.h"
#include "../fa_common.cuh"

#include <cstdint>
#include <vector>

namespace fa {
namespace ctc {

enum : int { kTimeMajor = 0, kVocabMajor = 1 };

struct TermDesc {
    int offset, count;   // the term's tokens in the flattened token array
    float norm;          // non-wildcard count, 1 when 0
    int pad;
};
struct ClipDesc {
    long long row0;       // first row of the clip in the concatenated log-probs
    long long cand0;      // first candidate slot of the clip's pairs
    int frames, cap;      // T and the candidate slots of each of its pairs
};
struct QueryDesc {
    long long start;      // clamped search start (row of the window's first frame)
    long long frames;     // clamped window length (may be <= 0)
    int offset, count;    // the query's tokens in the flattened token array
};
// The candidate slots a pair of a T-frame clip needs: at most ceil((T - N + 1) / 2) local maxima (no two are adjacent)
// or the one fallback, for any N >= 1.
inline int candidate_cap(int frames) { return frames / 2 + 2; }

int log_softmax(CallContext &C, bool on_device, const float *logits, int frames, int vocab, int layout,
                float temperature, float blank_bias, int blank_id, float *log_probs);
// rows: for each output row its source rows (CSR over src); the host has planned them from the chunk offsets
int merge_chunks(CallContext &C, bool on_device, const float *chunks, long long in_rows, int vocab,
                 const std::vector<long long> &row_src, const std::vector<long long> &src, float *out);
int spot_constrained(CallContext &C, bool on_device, const float *log_probs, int frames, int vocab, int blank_id,
                     const std::vector<QueryDesc> &queries, const std::vector<int> &tokens, float *score,
                     int64_t *start_frame, int64_t *end_frame);

// The vocabulary of fa_ctc_spotter in HBM, with its stream and buffers.
struct Spotter {
    int device = 0;
    Stream stream;   // declared first, so destroyed last
    int vocab = 0, blank_id = 0, terms = 0;
    std::vector<int> term_len;
    DeviceBuffer<> d_terms;      // TermDesc [K] then tokens
    DeviceBuffer<> d_buf;        // one host-buffer call's inputs and outputs
    DeviceBuffer<> scratch;      // candidates and per-pair counts
    UploadStage<> stage;         // clip descriptors, thresholds, detection offsets
    PinnedBuffer<int> h_counts;

    int init(int vocab, int blank_id, int terms, const int32_t *tokens, const int64_t *offsets);
    int spot(bool on_device, const float *log_probs, const int64_t *row_offsets, int clips, const float *min_score,
             int64_t *counts, int64_t *total, fa_ctc_detection *detections, long long capacity);
};

} // namespace ctc
} // namespace fa
