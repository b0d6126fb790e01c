// Sortformer streaming state in HBM (fa_sortformer_*): host bookkeeping (sortformer_streams.cu) and the two kernels'
// launchers (sortformer_kernels.cu).  Arithmetic: sortformer_core.cuh.
#pragma once

#include "fa_common.cuh"
#include "session_table.h"
#include "sortformer_core.cuh"

namespace fa {
namespace sortformer {

// One session's advance in a push, planned on the host from lengths alone (SortformerStateUpdater.swift:31-165).
struct Step {
    int core;            // coreFrames
    int pop;             // popOutLength, 0 when the FIFO does not overflow
    int compress;        // the speaker cache overflows after the pop
    int init_preds;      // first compression: spkcachePreds = preds[0, spkcacheLength) + popped rows (:151-158)
    int spkcache_after, fifo_after, has_preds_after;
};

// Checks and plans one update of a session with the given lengths; FA_INVALID_ARGUMENT (error text set) when the
// reference throws, coreFrames is negative or above max_core, or a context is negative.
int plan_step(const Config &c, int spkcache_len, int fifo_len, int has_preds, int emb_length, long long pred_rows, int lc,
              int rc, Step &out);

// The reference init's clamps (SortformerTypes.swift:239-254) and the checks create applies.
int resolve_config(const Config &in, int max_core, Config &out);

// Per-session descriptor of an update push (one CTA each).
struct UpdateJob {
    long long state;     // float offset of the session's arena
    long long silence;   // index of its silence count
    long long emb, pred; // float offsets of its batch row in chunk_embs / preds
    long long confirmed, tentative;   // float offsets of its output rows
    int spk_len, fifo_len, fifo_head, parity;
    int lc, rc, core, pop, compress, init_preds;
};

// Per-session descriptor of a model-input gather.
struct InputJob {
    long long state;
    int spk_len, fifo_len, fifo_head, parity;
};

// A session's arena, in floats from its offset: FIFO ring [fifo_rows x 512], its predictions [fifo_rows x 4], two
// speaker caches [cache_rows x 512] and their predictions [cache_rows x 4] (ping-pong for the compression's gather),
// the silence mean [512].  Each part starts 16-byte aligned.
struct Arena {
    long long fifo, fifo_preds, cache[2], cache_preds[2], mean, stride;
    void init(const Config &c);
    FA_HD long long cache_at(int b) const { return b ? cache[1] : cache[0]; }   // no local-memory indexing in kernels
    FA_HD long long cache_preds_at(int b) const { return b ? cache_preds[1] : cache_preds[0]; }
};

int launch_update(const Config &c, const Arena &a, const UpdateJob *d_jobs, int count, const float *embs, const float *preds,
                  float *state, long long *silence, float *confirmed, float *tentative, cudaStream_t s);
int launch_inputs(const Config &c, const Arena &a, const InputJob *d_jobs, int count, const float *state, float *spkcache,
                  float *fifo, cudaStream_t s);
size_t update_smem_bytes(const Config &c);
int set_update_smem(const Config &c);

struct SessionInfo {
    int spkcache_length, fifo_length, has_spkcache_preds, has_fifo_preds;
    long long chunks, silence_frames;
};

// A session's host mirror (sortformer_streams.cu): parity is the current cache buffer, chunks the updates so far.
struct SortformerSession {
    int spk_len, fifo_len, fifo_head, parity, has_preds;
    long long chunks;
};

class SortformerSet {
  public:
    Config cfg{};

    int init(const Config &resolved);
    int open(int *session);
    int close(int session);
    int update(int count, const int *sessions, const float *embs, int emb_rows, const float *preds, int pred_rows,
               const int *emb_lengths, const int *left, const int *right, bool device, float *confirmed,
               long long confirmed_len, float *tentative, long long tentative_len, int64_t *confirmed_rows,
               int64_t *tentative_rows);
    int model_inputs(int count, const int *sessions, bool device, float *spkcache, float *fifo, int *spkcache_lengths,
                     int *fifo_lengths);
    int state(int session, SessionInfo *info, float *spkcache, float *spkcache_preds, float *fifo, float *fifo_preds,
              float *mean);

  private:
    Arena arena{};
    Stream stream;
    SessionTable<SortformerSession> table;
    DeviceBuffer<float> d_state;
    DeviceBuffer<long long> d_silence;
    UploadStage<> update_desc, input_desc;
    DeviceBuffer<> staging;   // the host-buffer variants' arrays (HostStaging, fa_common.cuh)
};

} // namespace sortformer
} // namespace fa
