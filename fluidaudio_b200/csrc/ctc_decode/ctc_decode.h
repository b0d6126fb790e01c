// Host side of CTC decoding (ctc_decode_kernels.cu), behind the C ABI of ctc_decode_abi.cu.  Arguments reach these
// functions already checked; each returns an FA_* status.
#pragma once

#include "../../../include/fluidaudio_b200_ctc_decode.h"
#include "../call_context.h"
#include "../fa_common.cuh"
#include "ctc_decode_core.cuh"

#include <cstdint>
#include <vector>

namespace fa {
namespace ctc_decode {

struct ClipDesc {
    long long row0;    // first row of the clip in the concatenated log-probs (and of its staged tokens)
    long long node0;   // first slot of the clip's prefix trie
    long long cap;     // its slots: 2 * T * B + 1
    int frames, pad;
};

// The host copy of an LM before upload: checked by the C ABI.
struct LmTables {
    std::vector<unsigned long long> child_key, bigram_key;
    std::vector<int> child_node, node_word;
    std::vector<float> uni_log_prob, uni_backoff, bigram_log_prob;
};

// An ARPALanguageModel in HBM (fa_ctc_lm): read-only once made.
struct Lm {
    int device = 0;
    Stream stream;   // the upload's; declared first, so destroyed last
    DeviceBuffer<> d;
    LmView view{};                 // device pointers, on the host
    const LmView *d_view = nullptr;   // the same in HBM, for the kernels

    int init(const LmTables &t);
};

// fa_ctc_decoder: the piece table in HBM, with the stream and buffers of its calls.
struct Decoder {
    int device = 0;
    Stream stream;   // declared first, so destroyed last
    int vocab = 0, blank_id = 0;
    DeviceBuffer<> d_pieces;   // offsets [V + 1], boundary flags [V], bytes
    Pieces pieces{};
    DeviceBuffer<> d_buf;      // one host-buffer call's inputs and outputs
    DeviceBuffer<> scratch;    // top-K, prefix tries, staged tokens, per-clip results
    UploadStage<> stage;       // clip descriptors, then the output offsets
    PinnedBuffer<> h_res;      // per-clip lengths and scores, and the refusal flag

    int init(int vocab, int blank_id, const char *pieces, const int64_t *offsets);
    int beam_search(const Lm *lm, bool on_device, const float *log_probs, const int64_t *row_offsets, int clips,
                    int beam_width, int k_eff, float lm_weight, float word_bonus, int64_t *lengths, float *scores,
                    int32_t *tokens, long long capacity, int64_t *total);
};

// ctcGreedyDecode for many clips on a leased call context
int greedy(CallContext &C, bool on_device, const float *log_probs, const int64_t *row_offsets, int clips, int vocab,
           int blank_id, int64_t *lengths, int32_t *tokens, long long capacity, int64_t *total);

} // namespace ctc_decode
} // namespace fa
