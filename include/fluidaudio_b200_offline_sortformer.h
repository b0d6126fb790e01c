/* Offline Sortformer diarization around the caller's model (Sources/FluidAudio/Diarizer/Sortformer/Offline/
 * OfflineSortformerDiarizer.swift:279-375 with SortformerSpeakerStitcher.swift): the work processComplete does between
 * the log-mel and the timeline, for every window of many files per launch.  The fused mel -> speaker_preds model stays
 * with the caller.
 *
 * A file's life, one call each (no file outlives a call, so there is no handle):
 *   fa_mel_compute_batch[_device]            its time-major log-mel rows (default AudioMelSpectrogram, 128 mels)
 *   fa_offline_sortformer_plan               its window count and output rows
 *   fa_offline_sortformer_model_inputs       every window's channels-first mel and mel_length, all files in one batch
 *   (the caller's model)                     speaker_preds [windows x 384 x 4]
 *   fa_offline_sortformer_stitch             the windows' speaker columns aligned and averaged into one timeline
 *   fa_diarizer_timeline_push[_device]       those rows as finalized rows (finalized_rows = output_frames), then
 *   + fa_diarizer_timeline_finalize          finalize: rebuild(..., isComplete: true) on a fresh session
 * processComplete runs the model, then stitches, window by window; no window's model input depends on a stitch, so
 * every window of every file can go to the model as one batch and be stitched afterwards, with the same result.
 *
 * The only knob is overlapOutputFrames: every call takes `overlap` and clamps it as processComplete does, to
 * max(0, min(overlap, 383)); it is never refused.  hopOut = 384 - overlap and hopMel = 8 hopOut.  A file of n mel
 * frames (0 .. 2^40) has totalOut = ceil(n / 8) output rows; window k starts at mel frame k hopMel with
 * validMel = min(3072, n - k hopMel) frames and validOut = ceil(validMel / 8) rows, and the windows run while their
 * start is inside the file, ending after the first window with validMel < 3072.  0 frames is 0 windows and 0 rows: the
 * reference's empty timeline.  Windows are file-major, in window order, in every array.
 *
 * Every data-taking call has a host variant, which returns after its synchronisation, and a _device variant, whose
 * bulk arrays (mappings included) are HBM and which is asynchronous on the library's pooled call stream.  mel_offsets
 * and mel_frames stay host arrays.  Every call checks every argument
 * before any copy or launch, and a refused call writes nothing.  Launch counts are given for at least one window.
 *
 * Arithmetic (DESIGN §4.16), bit for bit with the reference's Swift (which does not contract), denormals kept:
 *   correlation  c[g][w] = c[g][w] + gv * wv in float32 over the overlap frames in ascending order, the product and the
 *                sum rounded separately, a frame skipped for row g when gv == 0 (+0 and -0; NaN is not skipped).
 *   score        (((0 + c[0][p0]) + c[1][p1]) + c[2][p2]) + c[3][p3] in float32.
 *   choice       the permutations in the stitcher's swap-recursion order (0123, 0132, 0213, 0231, 0321, 0312, 1023,
 *                ...); the first whose score is strictly greater than the best so far, which starts at -FLT_MAX.  NaN
 *                and -inf never win, +0 and -0 tie (the first keeps the lead), and identity results when nothing beats
 *                -FLT_MAX.  mapping[w] = g inverts the winner perm[g] = w.
 *   writing      a frame some earlier window of the file wrote becomes (global + pred) * 0.5f, the add then the
 *                multiply rounded; a new frame becomes pred.  Each window averages in turn, in window order.
 */
#ifndef FLUIDAUDIO_B200_OFFLINE_SORTFORMER_H
#define FLUIDAUDIO_B200_OFFLINE_SORTFORMER_H

#include "fluidaudio_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define FA_OFFLINE_SORTFORMER_WINDOW_OUT 384       /* OfflineSortformerConfig.windowOutputFrames */
#define FA_OFFLINE_SORTFORMER_SUBSAMPLING 8        /* subsamplingFactor */
#define FA_OFFLINE_SORTFORMER_WINDOW_MEL 3072      /* windowMelFrames = 384 * 8 */
#define FA_OFFLINE_SORTFORMER_SPEAKERS 4           /* numSpeakers */
#define FA_OFFLINE_SORTFORMER_MELS 128             /* melFeatures */
#define FA_OFFLINE_SORTFORMER_DEFAULT_OVERLAP 100  /* overlapOutputFrames' default */
/* frameDurationSeconds: Float(8) * Float(160) / Float(16000) = 0.08f, the float32 nearest 0.08 */

/* For `count` files of mel_frames[i] mel frames: window_counts[i] and output_frames[i] = ceil(mel_frames[i] / 8).  A
 * negative frame count, or one above 2^40, is FA_STATUS_INVALID_ARGUMENT with nothing written.  No device. */
fa_status fa_offline_sortformer_plan(int32_t overlap, int32_t count, const int64_t *mel_frames, int64_t *window_counts,
                                     int64_t *output_frames);

/* runOffline's copy (:98-119) for every window of `count` files.  File i's time-major rows [mel_frames[i] x 128] start
 * at mel + mel_offsets[i] (the out_offsets and num_frames fa_mel_compute_batch[_device] returns).  For W = the sum of
 * the files' window counts (at most window_capacity, else FA_STATUS_OUTPUT_TOO_SMALL), writes
 *   model_mel   [W x 128 x 3072]  channels-first: channel c, frame t < validMel is mel row melStart + t, then +0
 *   mel_length  [W] int32         validMel
 * W is at most 2^24.  1 launch. */
fa_status fa_offline_sortformer_model_inputs(int32_t overlap, int32_t count, const float *mel,
                                             const int64_t *mel_offsets, const int64_t *mel_frames,
                                             int64_t window_capacity, float *model_mel, int32_t *mel_length);
fa_status fa_offline_sortformer_model_inputs_device(int32_t overlap, int32_t count, const float *d_mel,
                                                    const int64_t *mel_offsets, const int64_t *mel_frames,
                                                    int64_t window_capacity, float *d_model_mel,
                                                    int32_t *d_mel_length);

/* processComplete's stitching for `count` files: speaker_preds [W x 384 x 4] is the model's output for the windows
 * fa_offline_sortformer_model_inputs wrote (only rows < validOut of a window are read).  Writes
 *   predictions  [sum of output_frames x 4]  packed in file order: the finalized rows fa_diarizer_timeline_push[_device]
 *                                            takes, with finalized_rows = output_frames
 *   mappings     [W x 4] int32 or NULL       each window's mapping[w] = g (identity for a file's first window)
 * One warp per file walks its windows in order; the files run in parallel.  1 launch. */
fa_status fa_offline_sortformer_stitch(int32_t overlap, int32_t count, const int64_t *mel_frames,
                                       const float *speaker_preds, float *predictions, int32_t *mappings);
fa_status fa_offline_sortformer_stitch_device(int32_t overlap, int32_t count, const int64_t *mel_frames,
                                              const float *d_speaker_preds, float *d_predictions, int32_t *d_mappings);

#ifdef __cplusplus
}
#endif

#endif /* FLUIDAUDIO_B200_OFFLINE_SORTFORMER_H */
