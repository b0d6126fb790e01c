// Host interface of the offline diarizer's prepare stage (prepare_kernels.cu): what OfflineDiarizerManager.prepare computes
// between the segmentation network and the embedding network, and between the embedding network and cluster(_:).
//
// Reference: Diarizer/Offline/Segmentation/OfflineSegmentationProcessor.swift (windows :55-56,118-187,190,303; decoding
// :321-405), Diarizer/Offline/Extraction/OfflineEmbeddingExtractor.swift (chunks and fbank windows :651-707; masks
// :421-613; the mask-similarity skip strategy :338-351,554-585,632-639), Extraction/WeightInterpolation.swift.
//
// Every call runs on the stream of the call context it is given and has finished when it returns; the host-buffer calls
// stage their arrays in the context's workspace `d_buf` (HostStaging, fa_common.cuh).  `on_device` says whether the large buffers (audio, windows, logits,
// log-probabilities, weights, the per-entry outputs) are device pointers; the small ones (chunk offsets, chunk indices,
// histogram, counts) are always host memory.
#pragma once

#include <cstdint>

namespace fa {
struct CallContext;   // call_context.h

namespace prepare {

constexpr int kMaxClasses = 16;   // logits per frame fa_seg_decode accepts

struct SegConfig {
    int sample_rate = 16000;
    double window_duration = 10.0;
    double step_ratio = 0.2;
    float speech_onset_threshold = 0.5f;
};

struct PlanConfig {
    bool exclude_overlap = true;
    double min_segment_duration = 1.0;
    float skip_threshold = -1.0f;     // < 0 (or NaN): EmbeddingSkipStrategy.none
    int weight_frames = 589;          // weightFrameCount
    int audio_sample_count = 160000;  // audioSampleCount
    int fbank_batch = 32;             // min(modelBatchLimit, 32)
};

struct WindowDesc {   // one gathered row: `copy` samples from audio[start], zeros after them
    long long start;
    long long copy;
};

struct PlanOutputs {  // per emitted entry, capacity chunks * speakers each; any pointer may be null
    int32_t *chunk_index, *speaker_index, *start_frame, *end_frame;
    double *start_time, *end_time;
    float *mask_sum;
    int32_t *used_fallback, *reuse_of;
    float *frame_weights;   // [entries x frames]         TimedEmbedding.frameWeights (maskToUse)
    float *model_weights;   // [entries x weight_frames]  the embedding network's weights input
};

bool seg_config_ok(const SegConfig &c);
long long samples_per_window(const SegConfig &c);   // OfflineDiarizerConfig.samplesPerWindow
long long samples_per_step(const SegConfig &c);     // .samplesPerStep
long long window_count(long long total_samples, const SegConfig &c);

// chunkOffsetSeconds of chunk c (:658-661) and its fbank window (:663-668, 819): copy == 0 when the chunk has no audio.
double resolve_chunk_offset(const double *offsets, int offsets_count, int c, const SegConfig &cfg);
WindowDesc embed_window(double chunk_offset, long long total_samples, const SegConfig &cfg, int audio_sample_count);

int gather_windows(CallContext &C, bool on_device, const float *audio, long long total_samples, const WindowDesc *desc,
                   int count, long long row_len, float *out);
int seg_decode(CallContext &C, bool on_device, const float *logits, int chunks, int frames, int classes, float onset,
               float *log_probs, float *speaker_weights, int64_t histogram[8], int64_t *speech_frames);
// counters: evaluatedMaskCount, emptyMaskCount, fallbackMaskCount, skippedEmbeddingCount
int embedding_plan(CallContext &C, bool on_device, const float *speaker_weights, int chunks, int frames, int speakers,
                   const double *chunk_offsets, int offsets_count, double frame_duration, long long total_samples,
                   const SegConfig &seg, const PlanConfig &plan, const PlanOutputs &out, int32_t *entry_count,
                   int64_t counters[4]);
int weight_resample(CallContext &C, const float *rows, long long row_count, int in_len, int out_len, float *out);

} // namespace prepare
} // namespace fa
