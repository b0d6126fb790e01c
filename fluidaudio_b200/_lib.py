"""ctypes binding of ``lib/libfluidaudio_b200.so`` (C ABI declared in ``include/fluidaudio_b200.h``,
``include/fluidaudio_b200_lseend.h``, ``include/fluidaudio_b200_ctc.h``, ``include/fluidaudio_b200_ctc_decode.h`` and
``include/fluidaudio_b200_vad.h``).

The library is the product: it is built in-tree by ``__graft_entry__.build()`` / ``make -C fluidaudio_b200/csrc``.
There is no Python or CPU fallback — if the shared object is missing, or no sm_90a device is visible, every
compute entry point raises.  This module never imports anything from ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libfluidaudio_b200.so")

STATUS_NAMES = {
    0: "OK", 1: "INVALID_ARGUMENT", 2: "INDEX_OVERFLOW", 3: "OUTPUT_TOO_SMALL", 4: "ALLOCATION_FAILURE",
    5: "RUNTIME_ERROR", 6: "NO_DEVICE", 7: "CUDA_ERROR", 8: "UNSUPPORTED", 255: "UNKNOWN_ERROR",
}


class FluidAudioError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        super().__init__(f"{where}: {STATUS_NAMES.get(status, status)}" + (f" — {detail}" if detail else ""))


NO_VALUE = -2 ** 31   # FA_NO_VALUE: an absent optional count (Swift nil)


class MelConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("n_mels", C.c_int32), ("n_fft", C.c_int32), ("hop_length", C.c_int32),
                ("win_length", C.c_int32), ("preemph", C.c_float), ("pad_to", C.c_int32), ("log_floor", C.c_float),
                ("log_floor_mode", C.c_int32), ("window_periodic", C.c_int32)]


class MelExConfig(C.Structure):
    _fields_ = [("base", MelConfig), ("filterbank", C.c_int32), ("filter_sample_rate", C.c_int32), ("f_min", C.c_float),
                ("f_max", C.c_float), ("center_edge", C.c_int32), ("spectrum_power", C.c_float),
                ("log_mean", C.c_float), ("log_std", C.c_float)]


class AudioFormat(C.Structure):
    _fields_ = [("in_rate", C.c_double), ("out_rate", C.c_double), ("channels", C.c_int32), ("format", C.c_int32),
                ("interleaved", C.c_int32), ("algorithm", C.c_int32)]


class VbxConfig(C.Structure):
    _fields_ = [("Fa", C.c_double), ("Fb", C.c_double), ("max_iterations", C.c_int32), ("epsilon", C.c_double),
                ("init_smoothing", C.c_double)]


class ClusterConfig(C.Structure):
    _fields_ = [("threshold", C.c_double), ("vbx", VbxConfig), ("num_speakers", C.c_int32),
                ("min_speakers", C.c_int32), ("max_speakers", C.c_int32), ("reserved", C.c_int32)]


class ClusterInfo(C.Structure):
    _fields_ = [("training_count", C.c_int32), ("initial_clusters", C.c_int32), ("vbx_iterations", C.c_int32),
                ("centroid_count", C.c_int32), ("ms_normalize", C.c_float), ("ms_ahc", C.c_float),
                ("ms_cut", C.c_float), ("ms_vbx", C.c_float), ("ms_assign", C.c_float), ("ms_total", C.c_float),
                ("was_adjusted", C.c_int32), ("detected_clusters", C.c_int32)]


class ReconstructConfig(C.Structure):
    _fields_ = [("frame_duration", C.c_double), ("window_duration", C.c_double), ("min_gap_duration", C.c_double),
                ("seg_min_duration_off", C.c_double), ("seg_min_duration_on", C.c_double),
                ("min_segment_duration", C.c_double), ("exclusive_segments", C.c_int32), ("reserved", C.c_int32)]


class SegConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("speech_onset_threshold", C.c_float), ("window_duration", C.c_double),
                ("step_ratio", C.c_double)]


class EmbedPlanConfig(C.Structure):
    _fields_ = [("exclude_overlap", C.c_int32), ("skip_threshold", C.c_float), ("min_segment_duration", C.c_double),
                ("weight_frames", C.c_int32), ("audio_sample_count", C.c_int32), ("fbank_batch", C.c_int32),
                ("reserved", C.c_int32)]


class SortformerConfig(C.Structure):
    _fields_ = [("chunk_len", C.c_int32), ("chunk_left_context", C.c_int32), ("chunk_right_context", C.c_int32),
                ("fifo_len", C.c_int32), ("spkcache_len", C.c_int32), ("spkcache_update_period", C.c_int32),
                ("spkcache_sil_frames_per_spk", C.c_int32), ("silence_threshold", C.c_float),
                ("pred_score_threshold", C.c_float), ("scores_boost_latest", C.c_float), ("strong_boost_rate", C.c_float),
                ("weak_boost_rate", C.c_float), ("min_pos_scores_rate", C.c_float)]


class SortformerSessionInfo(C.Structure):
    _fields_ = [("spkcache_length", C.c_int32), ("fifo_length", C.c_int32), ("has_spkcache_preds", C.c_int32),
                ("has_fifo_preds", C.c_int32), ("chunks", C.c_int64), ("silence_frames", C.c_int64)]


class TimelineConfig(C.Structure):
    _fields_ = [("num_speakers", C.c_int32), ("frame_duration_seconds", C.c_float), ("onset_threshold", C.c_float),
                ("offset_threshold", C.c_float), ("onset_pad_frames", C.c_int32), ("offset_pad_frames", C.c_int32),
                ("min_frames_on", C.c_int32), ("min_frames_off", C.c_int32), ("activity_type", C.c_int32),
                ("max_stored_frames", C.c_int32)]


class TimelineScratch(C.Structure):
    _fields_ = [("start_frame", C.c_int64), ("end_frame", C.c_int64), ("unmerged_start_frame", C.c_int64),
                ("active_frame_count", C.c_int64), ("unmerged_active_frame_count", C.c_int64),
                ("activity_sum", C.c_float), ("unmerged_activity_sum", C.c_float), ("speaking", C.c_int32),
                ("has_segment", C.c_int32)]


class TimelineSessionInfo(C.Structure):
    _fields_ = [("finalized_frames", C.c_int64), ("stored_frames", C.c_int64), ("tentative_frames", C.c_int64)]


class LSEENDStreamConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("n_mels", C.c_int32), ("hop_length", C.c_int32), ("win_length", C.c_int32),
                ("context_size", C.c_int32), ("subsampling", C.c_int32), ("chunk_size", C.c_int32),
                ("conv_delay", C.c_int32), ("precision", C.c_int32)]


class LSEENDStreamSizes(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("n_fft", "mel_frames", "chunk_mels", "mel_context", "chunk_samples",
                                         "audio_left_context", "audio_context", "flush_samples", "mask_length",
                                         "audio_capacity")]


class LSEENDSessionInfo(C.Structure):
    _fields_ = [("audio_samples", C.c_int64), ("mel_rows", C.c_int64), ("cmn_count", C.c_int64),
                ("decoder_mask_end", C.c_int32), ("has_snapshot", C.c_int32)]


class CtcDetection(C.Structure):
    _fields_ = [("clip", C.c_int32), ("term", C.c_int32), ("score", C.c_float), ("start_frame", C.c_int32),
                ("end_frame", C.c_int32)]


class CtcBeamConfig(C.Structure):
    _fields_ = [("beam_width", C.c_int32), ("token_candidates", C.c_int32), ("lm_weight", C.c_float),
                ("word_bonus", C.c_float)]


class VadConfig(C.Structure):
    _fields_ = [("default_threshold", C.c_float), ("min_speech_duration", C.c_double),
                ("min_silence_duration", C.c_double), ("max_speech_duration", C.c_double),
                ("speech_padding", C.c_double), ("silence_threshold_for_split", C.c_float),
                ("has_negative_threshold", C.c_int32), ("negative_threshold", C.c_float),
                ("negative_threshold_offset", C.c_float), ("min_silence_at_max_speech", C.c_double),
                ("use_max_possible_silence_at_max_speech", C.c_int32)]


class VadResolved(C.Structure):
    _fields_ = [("threshold", C.c_float), ("negative_threshold", C.c_float),
                ("silence_threshold_for_split", C.c_float), ("use_max_possible_silence_at_max_speech", C.c_int32),
                ("min_speech_samples", C.c_int64), ("min_silence_samples", C.c_int64),
                ("max_speech_samples", C.c_int64), ("speech_pad_samples", C.c_int64),
                ("min_silence_at_max_speech_samples", C.c_int64)]


class VadSessionInfo(C.Structure):
    _fields_ = [("triggered", C.c_int32), ("has_pending", C.c_int32), ("temp_end_sample", C.c_int64),
                ("processed_samples", C.c_int64)]


# fa_ctc_detection as a numpy record
CTC_DETECTION = np.dtype([("clip", np.int32), ("term", np.int32), ("score", np.float32), ("start_frame", np.int32),
                          ("end_frame", np.int32)])

# fa_diarizer_timeline_segment as a numpy record
TIMELINE_SEGMENT = np.dtype([("start_frame", np.int64), ("end_frame", np.int64), ("activity", np.float32),
                             ("speaker", np.int32)])


# every symbol include/fluidaudio_b200.h and include/FastClusterWrapper.h declare (tests check the export table)
EXPORTED_SYMBOLS = [
    "fa_version", "fa_last_error", "fa_device_count", "fa_set_device", "fa_device_synchronize",
    "fa_kernel_launch_count", "fa_host_alloc", "fa_host_free", "fa_device_alloc", "fa_device_free", "fa_memcpy_h2d",
    "fa_memcpy_d2h", "fa_memcpy_probe", "fa_timer_start", "fa_timer_stop_ms", "fa_mel_default_config", "fa_mel_create",
    "fa_mel_destroy", "fa_mel_get_window", "fa_mel_get_filterbank", "fa_mel_frame_count", "fa_mel_compute",
    "fa_mel_compute_device", "fa_mel_compute_batch", "fa_mel_compute_batch_device", "fa_mel_timer_start",
    "fa_mel_timer_stop_ms", "fa_mel_set_precision", "fa_mel_get_precision", "fa_mel_set_pipeline_chunks", "fa_mel_set_zero_copy_output", "fa_mel_normalize_per_feature", "fa_mel_unified_features", "fa_mel_lseend_features",
    "fa_mel_ex_default_config", "fa_mel_preset_cohere", "fa_mel_preset_styletts2", "fa_mel_preset_luxtts",
    "fa_mel_create_ex", "fa_mel_cohere_features", "fa_mel_styletts2_features", "fa_mel_luxtts_features",
    "fa_mel_stream_open", "fa_mel_stream_close", "fa_mel_stream_frames", "fa_mel_stream_push", "fa_mel_stream_push_device",
    "fa_resample_output_count", "fa_audio_resample", "fa_audio_to_mel",
    "fa_linear_resample", "fa_l2_normalize_rows", "fa_ahc_cluster", "fa_dendrogram_cut", "fa_vbx_default_config",
    "fa_vbx_refine", "fa_compute_centroids", "fa_assign_embeddings", "fa_cluster_default_config",
    "fa_diarize_cluster", "fa_diarize_cluster_batch", "fa_diarize_cluster_batch_chunks", "fa_ahc_last_stage_ms", "fa_diarize_cluster_chunks",
    "fa_hungarian_solve", "fa_max_score_assignment", "fa_constrained_assign", "fa_build_chunk_assignments",
    "fa_export_shape", "fa_export_read", "fa_export_write", "fa_kmeans_cluster", "fa_speaker_constraints_resolve",
    "fa_reconstruct_default_config", "fa_build_segments", "fa_build_speaker_database",
    "fa_seg_default_config", "fa_embed_plan_default_config", "fa_seg_window_count", "fa_seg_windows",
    "fa_seg_windows_device", "fa_seg_decode", "fa_seg_decode_device", "fa_embedding_plan", "fa_embedding_plan_device",
    "fa_embed_windows", "fa_embed_windows_device", "fa_weight_resample",
    "fa_sortformer_default_config", "fa_sortformer_resolve_config", "fa_sortformer_step", "fa_sortformer_create",
    "fa_sortformer_destroy", "fa_sortformer_open", "fa_sortformer_close", "fa_sortformer_update",
    "fa_sortformer_update_device", "fa_sortformer_model_inputs", "fa_sortformer_model_inputs_device",
    "fa_sortformer_session_state",
    "fa_diarizer_timeline_default_config", "fa_diarizer_timeline_config_from_seconds",
    "fa_diarizer_timeline_segment_bound", "fa_diarizer_timeline_create", "fa_diarizer_timeline_destroy",
    "fa_diarizer_timeline_open", "fa_diarizer_timeline_close", "fa_diarizer_timeline_push",
    "fa_diarizer_timeline_push_device", "fa_diarizer_timeline_finalize", "fa_diarizer_timeline_reset",
    "fa_diarizer_timeline_clear_speaker", "fa_diarizer_timeline_session_state",
    "fastcluster_compute_centroid_linkage",
]

# every symbol include/fluidaudio_b200_lseend.h declares (the LS-EEND feature streams)
LSEEND_SYMBOLS = [
    "fa_lseend_stream_resolve", "fa_lseend_stream_create", "fa_lseend_stream_destroy", "fa_lseend_stream_open",
    "fa_lseend_stream_close", "fa_lseend_stream_chunks", "fa_lseend_stream_push", "fa_lseend_stream_push_device",
    "fa_lseend_stream_snapshot", "fa_lseend_stream_rollback", "fa_lseend_stream_reset",
    "fa_lseend_stream_session_state",
]

# every symbol include/fluidaudio_b200_ctc.h declares (CTC keyword spotting)
CTC_SYMBOLS = [
    "fa_ctc_log_softmax", "fa_ctc_log_softmax_device", "fa_ctc_merge_chunks", "fa_ctc_merge_chunks_device",
    "fa_ctc_spotter_create", "fa_ctc_spotter_destroy", "fa_ctc_spot", "fa_ctc_spot_device", "fa_ctc_spot_constrained",
    "fa_ctc_spot_constrained_device",
]

# every symbol include/fluidaudio_b200_ctc_decode.h declares (CTC decoding)
CTC_DECODE_SYMBOLS = [
    "fa_ctc_beam_default_config", "fa_ctc_lm_create", "fa_ctc_lm_destroy", "fa_ctc_decoder_create",
    "fa_ctc_decoder_destroy", "fa_ctc_beam_search", "fa_ctc_beam_search_device", "fa_ctc_greedy",
    "fa_ctc_greedy_device",
]

class OnlineDiarConfig(C.Structure):
    """fa_od_config's layout"""
    _fields_ = [("clustering_threshold", C.c_float), ("min_speech_duration", C.c_float),
                ("min_embedding_update_duration", C.c_float), ("min_silence_gap", C.c_float),
                ("num_clusters", C.c_int32), ("min_active_frames_count", C.c_float), ("chunk_duration", C.c_float),
                ("chunk_overlap", C.c_float)]


class OnlineDiarResolved(C.Structure):
    """fa_od_resolved's layout"""
    _fields_ = [("speaker_threshold", C.c_float), ("embedding_threshold", C.c_float),
                ("min_speech_duration", C.c_float), ("min_active_frames_count", C.c_float),
                ("chunk_size", C.c_int64), ("step_size", C.c_int64)]


ONLINE_DIAR_SPEAKER = np.dtype([("key", "<i8"), ("numeric", "<i8"), ("update_count", "<i8"), ("duration", "<f4"),
                                ("named", "<i4"), ("has_numeric", "<i4"), ("permanent", "<i4"),
                                ("raw_count", "<i4")], align=True)   # fa_od_speaker's layout


# every symbol include/fluidaudio_b200_vad.h declares (voice activity detection)
VAD_SYMBOLS = [
    "fa_vad_default_config", "fa_vad_resolve", "fa_vad_stream_create", "fa_vad_stream_destroy", "fa_vad_stream_open",
    "fa_vad_stream_close", "fa_vad_stream_model_inputs", "fa_vad_stream_model_inputs_device", "fa_vad_stream_advance",
    "fa_vad_stream_advance_device", "fa_vad_stream_session_state", "fa_vad_segment", "fa_vad_segment_device",
    "fa_fsmn_vad_decide", "fa_fsmn_vad_decide_device",
]

# every symbol include/fluidaudio_b200_online_diar.h declares (streaming speaker tracking)
ONLINE_DIAR_SYMBOLS = [
    "fa_od_default_config", "fa_od_resolve", "fa_od_chunk_inputs", "fa_od_chunk_inputs_device",
    "fa_od_enrollment_inputs", "fa_od_enrollment_inputs_device", "fa_od_create", "fa_od_destroy", "fa_od_open",
    "fa_od_close", "fa_od_embedding_inputs", "fa_od_embedding_inputs_device", "fa_od_advance", "fa_od_advance_device",
    "fa_od_query", "fa_od_query_device", "fa_od_speaker_count", "fa_od_read", "fa_od_initialize", "fa_od_remove",
    "fa_od_merge", "fa_od_set_permanent", "fa_od_reset", "fa_od_upsert",
]

# every symbol include/fluidaudio_b200_luxtts.h declares (LuxTTS synthesis around the caller's models)
LUXTTS_SYMBOLS = [
    "fa_luxtts_plan", "fa_luxtts_create", "fa_luxtts_destroy", "fa_luxtts_begin", "fa_luxtts_begin_device",
    "fa_luxtts_text_condition", "fa_luxtts_text_condition_device", "fa_luxtts_model_inputs",
    "fa_luxtts_model_inputs_device", "fa_luxtts_advance", "fa_luxtts_advance_device", "fa_luxtts_vocoder_input",
    "fa_luxtts_vocoder_input_device", "fa_luxtts_finish", "fa_luxtts_finish_device", "fa_luxtts_close",
    "fa_luxtts_request_state",
]


# every symbol include/fluidaudio_b200_styletts2.h declares (StyleTTS2 synthesis glue around the caller's models)
STYLETTS2_SYMBOLS = [
    "fa_styletts2_plan", "fa_styletts2_sampler_inputs", "fa_styletts2_sampler_inputs_device", "fa_styletts2_style",
    "fa_styletts2_style_device", "fa_styletts2_align", "fa_styletts2_align_device",
]


# every symbol include/fluidaudio_b200_offline_sortformer.h declares (offline Sortformer windows around the caller's
# model)
OFFLINE_SORTFORMER_SYMBOLS = [
    "fa_offline_sortformer_plan", "fa_offline_sortformer_model_inputs", "fa_offline_sortformer_model_inputs_device",
    "fa_offline_sortformer_stitch", "fa_offline_sortformer_stitch_device",
]


class LuxTtsPlanInfo(C.Structure):
    """fa_luxtts_plan_info's layout"""
    _fields_ = [("reason", C.c_int32), ("prompt_samples", C.c_int32), ("prompt_frames", C.c_int32),
                ("token_count", C.c_int32), ("features_length", C.c_int32), ("gen_frames", C.c_int32),
                ("bucket", C.c_int32), ("boosted", C.c_int32), ("prompt_rms", C.c_float), ("step", C.c_int32)]


_lib = None


def load():
    """Load the CUDA library, failing loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FluidAudioError(6, "fluidaudio_b200",
                              f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, f32, f64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double, C.c_size_t
    L.fa_version.restype = C.c_char_p
    L.fa_last_error.restype = C.c_char_p
    L.fa_device_count.restype = i32
    L.fa_set_device.argtypes = [i32]
    L.fa_kernel_launch_count.restype = i64
    L.fa_host_alloc.argtypes = [sz, C.POINTER(vp)]
    L.fa_host_free.argtypes = [vp]
    L.fa_device_alloc.argtypes = [sz, C.POINTER(vp)]
    L.fa_device_free.argtypes = [vp]
    L.fa_memcpy_h2d.argtypes = [vp, vp, sz]
    L.fa_memcpy_d2h.argtypes = [vp, vp, sz]
    L.fa_memcpy_probe.argtypes = [vp, sz, vp, sz, i32, C.POINTER(f32)]
    L.fa_timer_stop_ms.argtypes = [C.POINTER(f32)]
    L.fa_mel_default_config.argtypes = [C.POINTER(MelConfig)]
    L.fa_mel_default_config.restype = None
    L.fa_mel_create.argtypes = [C.POINTER(MelConfig), C.POINTER(vp)]
    for name in ("fa_mel_ex_default_config", "fa_mel_preset_cohere", "fa_mel_preset_styletts2", "fa_mel_preset_luxtts"):
        getattr(L, name).argtypes = [C.POINTER(MelExConfig)]
        getattr(L, name).restype = None
    L.fa_mel_create_ex.argtypes = [C.POINTER(MelExConfig), C.POINTER(vp)]
    L.fa_mel_cohere_features.argtypes = [vp, vp, sz, i64, vp, sz, C.POINTER(i64), C.POINTER(i64)]
    L.fa_mel_styletts2_features.argtypes = [vp, vp, sz, vp, sz, C.POINTER(i64)]
    L.fa_mel_luxtts_features.argtypes = [vp, vp, sz, vp, sz, C.POINTER(i64)]
    L.fa_mel_destroy.argtypes = [vp]
    L.fa_mel_destroy.restype = None
    L.fa_mel_get_window.argtypes = [vp, vp, sz]
    L.fa_mel_get_filterbank.argtypes = [vp, vp, sz]
    L.fa_mel_frame_count.argtypes = [vp, i64, i32, i64]
    L.fa_mel_frame_count.restype = i64
    L.fa_mel_compute.argtypes = [vp, vp, sz, f32, i32, i64, i32, vp, sz, C.POINTER(i64), C.POINTER(i64)]
    L.fa_mel_compute_device.argtypes = L.fa_mel_compute.argtypes
    L.fa_mel_compute_batch.argtypes = [vp, vp, vp, i32, vp, i32, i32, vp, vp, vp, vp]
    L.fa_mel_compute_batch_device.argtypes = L.fa_mel_compute_batch.argtypes
    L.fa_mel_set_precision.argtypes = [vp, i32]
    L.fa_mel_set_pipeline_chunks.argtypes = [vp, i32]
    L.fa_mel_set_zero_copy_output.argtypes = [vp, i32]
    L.fa_mel_get_precision.argtypes = [vp]
    L.fa_mel_get_precision.restype = i32
    L.fa_mel_timer_start.argtypes = [vp]
    L.fa_mel_timer_stop_ms.argtypes = [vp, C.POINTER(f32)]
    L.fa_mel_normalize_per_feature.argtypes = [vp, i64, i32, i64]
    L.fa_mel_unified_features.argtypes = [vp, vp, sz, sz, vp, sz, C.POINTER(i64), C.POINTER(i32)]
    L.fa_mel_lseend_features.argtypes = [vp, vp, sz, vp, C.POINTER(i64), vp, sz, C.POINTER(i64)]
    L.fa_mel_stream_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_mel_stream_close.argtypes = [vp, i32]
    L.fa_mel_stream_frames.argtypes = [vp, i32, i64, i32]
    L.fa_mel_stream_frames.restype = i64
    L.fa_mel_stream_push.argtypes = [vp, i32, vp, vp, vp, vp, vp, sz, vp]
    L.fa_mel_stream_push_device.argtypes = L.fa_mel_stream_push.argtypes
    L.fa_resample_output_count.argtypes = [C.POINTER(AudioFormat), i64]
    L.fa_resample_output_count.restype = i64
    L.fa_audio_resample.argtypes = [vp, i64, C.POINTER(AudioFormat), vp, i64, C.POINTER(i64)]
    L.fa_audio_to_mel.argtypes = [vp, vp, i64, C.POINTER(AudioFormat), f32, i32, i32, vp, sz, C.POINTER(i64),
                                  C.POINTER(i64), C.POINTER(i64)]
    L.fa_linear_resample.argtypes = [vp, i64, i32, f64, f64, vp, i64, C.POINTER(i64)]
    L.fa_l2_normalize_rows.argtypes = [vp, sz, sz, vp]
    L.fa_ahc_cluster.argtypes = [vp, sz, sz, f64, vp]
    L.fa_dendrogram_cut.argtypes = [vp, sz, f64, vp]
    L.fa_vbx_default_config.argtypes = [C.POINTER(VbxConfig)]
    L.fa_vbx_default_config.restype = None
    L.fa_vbx_refine.argtypes = [vp, sz, sz, vp, sz, vp, i32, C.POINTER(VbxConfig), vp, vp, vp, vp, C.POINTER(i32)]
    L.fa_compute_centroids.argtypes = [vp, sz, sz, vp, vp, i32, vp, C.POINTER(i32)]
    L.fa_assign_embeddings.argtypes = [vp, sz, sz, vp, i32, vp, vp]
    L.fa_cluster_default_config.argtypes = [C.POINTER(ClusterConfig)]
    L.fa_cluster_default_config.restype = None
    L.fa_diarize_cluster.argtypes = [vp, vp, sz, sz, sz, vp, C.POINTER(ClusterConfig), vp, vp, vp, i32,
                                     C.POINTER(ClusterInfo)]
    L.fa_diarize_cluster_batch.argtypes = [vp, vp, vp, i32, sz, sz, vp, C.POINTER(ClusterConfig), vp, vp]
    L.fa_diarize_cluster_batch_chunks.argtypes = [vp, vp, vp, i32, sz, sz, vp, C.POINTER(ClusterConfig), vp, vp, vp]
    L.fa_diarize_cluster_chunks.argtypes = [vp, vp, sz, sz, sz, vp, C.POINTER(ClusterConfig), vp, vp, vp, vp, i32,
                                            C.POINTER(ClusterInfo)]
    L.fa_hungarian_solve.argtypes = [vp, i32, vp]
    L.fa_max_score_assignment.argtypes = [vp, i32, i32, vp]
    L.fa_constrained_assign.argtypes = [vp, sz, i32, vp, vp]
    L.fa_build_chunk_assignments.argtypes = [vp, vp, vp, sz, i32, i32, i32, vp]
    L.fa_kmeans_cluster.argtypes = [vp, sz, sz, i32, i32, i32, C.c_uint64, vp, vp, i32, C.POINTER(i32), C.POINTER(i32)]
    L.fa_speaker_constraints_resolve.argtypes = [i64, i64, i64, i64, C.POINTER(i64), C.POINTER(i64)]
    L.fa_reconstruct_default_config.argtypes = [C.POINTER(ReconstructConfig)]
    L.fa_reconstruct_default_config.restype = None
    L.fa_build_segments.argtypes = [vp, i32, i32, i32, vp, i32, vp, i32, i32, C.POINTER(ReconstructConfig), vp, vp, vp, vp,
                                    i32, C.POINTER(i32)]
    L.fa_build_speaker_database.argtypes = [vp, i32, vp, i32, i32, vp, vp]
    L.fa_export_shape.argtypes = [C.c_char_p, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
    L.fa_export_read.argtypes = [C.c_char_p, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.fa_export_write.argtypes = [C.c_char_p, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.fa_seg_default_config.argtypes = [C.POINTER(SegConfig)]
    L.fa_seg_default_config.restype = None
    L.fa_embed_plan_default_config.argtypes = [C.POINTER(EmbedPlanConfig)]
    L.fa_embed_plan_default_config.restype = None
    L.fa_seg_window_count.argtypes = [i64, C.POINTER(SegConfig), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    L.fa_seg_windows.argtypes = [vp, i64, C.POINTER(SegConfig), i32, i32, vp, vp]
    L.fa_seg_windows_device.argtypes = L.fa_seg_windows.argtypes
    L.fa_seg_decode.argtypes = [vp, i32, i32, i32, C.POINTER(SegConfig), vp, vp, vp, C.POINTER(i64)]
    L.fa_seg_decode_device.argtypes = L.fa_seg_decode.argtypes
    L.fa_embedding_plan.argtypes = [vp, i32, i32, i32, vp, i32, f64, i64, C.POINTER(SegConfig),
                                    C.POINTER(EmbedPlanConfig)] + [vp] * 11 + [C.POINTER(i32), vp]
    L.fa_embedding_plan_device.argtypes = L.fa_embedding_plan.argtypes
    L.fa_embed_windows.argtypes = [vp, i64, vp, i32, vp, i32, C.POINTER(SegConfig), i32, vp]
    L.fa_embed_windows_device.argtypes = L.fa_embed_windows.argtypes
    L.fa_weight_resample.argtypes = [vp, i64, i32, i32, vp]
    SF = C.POINTER(SortformerConfig)
    L.fa_sortformer_default_config.argtypes = [SF, i32]
    L.fa_sortformer_resolve_config.argtypes = [SF, i32, SF, C.POINTER(i32)]
    L.fa_sortformer_step.argtypes = [SF, i32, vp, i32, i32, i32, i32, vp]
    L.fa_sortformer_create.argtypes = [SF, i32, C.POINTER(vp)]
    L.fa_sortformer_destroy.argtypes = [vp]
    L.fa_sortformer_destroy.restype = None
    L.fa_sortformer_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_sortformer_close.argtypes = [vp, i32]
    L.fa_sortformer_update.argtypes = [vp, i32, vp, vp, i32, vp, i32, vp, vp, vp, vp, sz, vp, sz, vp, vp]
    L.fa_sortformer_update_device.argtypes = L.fa_sortformer_update.argtypes
    L.fa_sortformer_model_inputs.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    L.fa_sortformer_model_inputs_device.argtypes = L.fa_sortformer_model_inputs.argtypes
    L.fa_sortformer_session_state.argtypes = [vp, i32, C.POINTER(SortformerSessionInfo), vp, vp, vp, vp, vp]
    TC = C.POINTER(TimelineConfig)
    L.fa_diarizer_timeline_default_config.argtypes = [TC, i32, i32, f32]
    L.fa_diarizer_timeline_config_from_seconds.argtypes = [TC, f32, f32, f32, f32]
    L.fa_diarizer_timeline_segment_bound.argtypes = [i32, i32, vp, vp, C.POINTER(i64), C.POINTER(i64)]
    L.fa_diarizer_timeline_create.argtypes = [TC, i32, C.POINTER(vp)]
    L.fa_diarizer_timeline_destroy.argtypes = [vp]
    L.fa_diarizer_timeline_destroy.restype = None
    L.fa_diarizer_timeline_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_diarizer_timeline_close.argtypes = [vp, i32]
    L.fa_diarizer_timeline_push.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, sz, vp, sz, vp, vp]
    L.fa_diarizer_timeline_push_device.argtypes = L.fa_diarizer_timeline_push.argtypes
    L.fa_diarizer_timeline_finalize.argtypes = [vp, i32, vp]
    L.fa_diarizer_timeline_reset.argtypes = [vp, i32, vp]
    L.fa_diarizer_timeline_clear_speaker.argtypes = [vp, i32, i32]
    L.fa_diarizer_timeline_session_state.argtypes = [vp, i32, C.POINTER(TimelineSessionInfo), vp, vp,
                                                     C.POINTER(TimelineScratch)]
    LC = C.POINTER(LSEENDStreamConfig)
    L.fa_lseend_stream_resolve.argtypes = [LC, C.POINTER(LSEENDStreamSizes)]
    L.fa_lseend_stream_create.argtypes = [LC, C.POINTER(vp)]
    L.fa_lseend_stream_destroy.argtypes = [vp]
    L.fa_lseend_stream_destroy.restype = None
    L.fa_lseend_stream_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_lseend_stream_close.argtypes = [vp, i32]
    L.fa_lseend_stream_chunks.argtypes = [vp, i32, i64, i32]
    L.fa_lseend_stream_chunks.restype = i64
    L.fa_lseend_stream_push.argtypes = [vp, i32, vp, vp, vp, vp, vp, sz, vp, sz, vp, sz, vp]
    L.fa_lseend_stream_push_device.argtypes = L.fa_lseend_stream_push.argtypes
    for name in ("fa_lseend_stream_snapshot", "fa_lseend_stream_rollback", "fa_lseend_stream_reset"):
        getattr(L, name).argtypes = [vp, i32, vp]
    L.fa_lseend_stream_session_state.argtypes = [vp, i32, C.POINTER(LSEENDSessionInfo), vp, vp, vp]
    L.fa_ctc_log_softmax.argtypes = [vp, i32, i32, i32, f32, f32, i32, vp]
    L.fa_ctc_log_softmax_device.argtypes = L.fa_ctc_log_softmax.argtypes
    L.fa_ctc_merge_chunks.argtypes = [vp, vp, i32, i32, i32, vp, sz, C.POINTER(i32)]
    L.fa_ctc_merge_chunks_device.argtypes = L.fa_ctc_merge_chunks.argtypes
    L.fa_ctc_spotter_create.argtypes = [i32, i32, i32, vp, vp, C.POINTER(vp)]
    L.fa_ctc_spotter_destroy.argtypes = [vp]
    L.fa_ctc_spotter_destroy.restype = None
    L.fa_ctc_spot.argtypes = [vp, vp, vp, i32, C.POINTER(f32), vp, C.POINTER(i64), vp, sz]
    L.fa_ctc_spot_device.argtypes = L.fa_ctc_spot.argtypes
    L.fa_ctc_spot_constrained.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]
    L.fa_ctc_spot_constrained_device.argtypes = L.fa_ctc_spot_constrained.argtypes
    L.fa_ctc_beam_default_config.argtypes = [C.POINTER(CtcBeamConfig)]
    L.fa_ctc_beam_default_config.restype = None
    L.fa_ctc_lm_create.argtypes = [i32, vp, vp, vp, vp, vp, i64, vp, vp, vp, C.POINTER(vp)]
    L.fa_ctc_lm_destroy.argtypes = [vp]
    L.fa_ctc_lm_destroy.restype = None
    L.fa_ctc_decoder_create.argtypes = [i32, i32, vp, vp, C.POINTER(vp)]
    L.fa_ctc_decoder_destroy.argtypes = [vp]
    L.fa_ctc_decoder_destroy.restype = None
    L.fa_ctc_beam_search.argtypes = [vp, vp, vp, vp, i32, C.POINTER(CtcBeamConfig), vp, vp, vp, sz, C.POINTER(i64)]
    L.fa_ctc_beam_search_device.argtypes = L.fa_ctc_beam_search.argtypes
    L.fa_ctc_greedy.argtypes = [vp, vp, i32, i32, i32, vp, vp, sz, C.POINTER(i64)]
    L.fa_ctc_greedy_device.argtypes = L.fa_ctc_greedy.argtypes
    VC = C.POINTER(VadConfig)
    L.fa_vad_default_config.argtypes = [VC]
    L.fa_vad_default_config.restype = None
    L.fa_vad_resolve.argtypes = [VC, C.POINTER(VadResolved)]
    L.fa_vad_stream_create.argtypes = [C.POINTER(vp)]
    L.fa_vad_stream_destroy.argtypes = [vp]
    L.fa_vad_stream_destroy.restype = None
    L.fa_vad_stream_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_vad_stream_close.argtypes = [vp, i32]
    L.fa_vad_stream_model_inputs.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]
    L.fa_vad_stream_model_inputs_device.argtypes = L.fa_vad_stream_model_inputs.argtypes
    L.fa_vad_stream_advance.argtypes = [vp, i32, vp, vp, vp, vp, VC, vp]
    L.fa_vad_stream_advance_device.argtypes = L.fa_vad_stream_advance.argtypes
    L.fa_vad_stream_session_state.argtypes = [vp, i32, C.POINTER(VadSessionInfo), vp, vp, vp]
    L.fa_vad_segment.argtypes = [vp, vp, i32, vp, VC, vp, vp, sz, C.POINTER(i64)]
    L.fa_vad_segment_device.argtypes = L.fa_vad_segment.argtypes
    L.fa_fsmn_vad_decide.argtypes = [vp, vp, i32, vp, vp, sz, C.POINTER(i64)]
    L.fa_fsmn_vad_decide_device.argtypes = L.fa_fsmn_vad_decide.argtypes
    OC = C.POINTER(OnlineDiarConfig)
    L.fa_od_default_config.argtypes = [OC]
    L.fa_od_default_config.restype = None
    L.fa_od_resolve.argtypes = [OC, C.POINTER(OnlineDiarResolved)]
    L.fa_od_chunk_inputs.argtypes = [vp, vp, i32, i64, vp, vp]
    L.fa_od_chunk_inputs_device.argtypes = L.fa_od_chunk_inputs.argtypes
    L.fa_od_enrollment_inputs.argtypes = [vp, vp, i32, i32, vp, vp]
    L.fa_od_enrollment_inputs_device.argtypes = L.fa_od_enrollment_inputs.argtypes
    L.fa_od_create.argtypes = [i32, C.POINTER(vp)]
    L.fa_od_destroy.argtypes = [vp]
    L.fa_od_destroy.restype = None
    L.fa_od_open.argtypes = [vp, C.POINTER(i32)]
    L.fa_od_close.argtypes = [vp, i32]
    L.fa_od_embedding_inputs.argtypes = [vp, i32, vp, vp, OC, vp, vp]
    L.fa_od_embedding_inputs_device.argtypes = L.fa_od_embedding_inputs.argtypes
    L.fa_od_advance.argtypes = [vp, i32, vp, vp, vp, OC, vp, vp, vp, vp]
    L.fa_od_advance_device.argtypes = L.fa_od_advance.argtypes
    L.fa_od_query.argtypes = [vp, i32, i32, vp, vp]
    L.fa_od_query_device.argtypes = L.fa_od_query.argtypes
    L.fa_od_speaker_count.argtypes = [vp, i32, C.POINTER(i64), C.POINTER(i64)]
    L.fa_od_read.argtypes = [vp, i32, vp, vp, vp]
    L.fa_od_initialize.argtypes = [vp, i32, i32, vp, vp, vp, i32, i32]
    L.fa_od_remove.argtypes = [vp, i32, i32, i64, i32, C.POINTER(i32)]
    L.fa_od_merge.argtypes = [vp, i32, i32, i64, i32, i64, i32, C.POINTER(i32)]
    L.fa_od_set_permanent.argtypes = [vp, i32, i32, i64, i32, C.POINTER(i32)]
    L.fa_od_reset.argtypes = [vp, i32, i32]
    L.fa_od_upsert.argtypes = [vp, i32, vp, vp, vp]
    L.fa_ahc_last_stage_ms.argtypes = [vp]
    L.fa_ahc_last_stage_ms.restype = None
    L.fastcluster_compute_centroid_linkage.argtypes = [vp, sz, sz, vp, sz]
    L.fastcluster_compute_centroid_linkage.restype = C.c_int
    LP = C.POINTER(LuxTtsPlanInfo)
    L.fa_luxtts_plan.argtypes = [i64, i32, i32, f32, LP]
    L.fa_luxtts_create.argtypes = [C.POINTER(vp)]
    L.fa_luxtts_destroy.argtypes = [vp]
    L.fa_luxtts_destroy.restype = None
    for name in ("fa_luxtts_begin", "fa_luxtts_begin_device"):
        getattr(L, name).argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, LP, vp, vp]
    for name in ("fa_luxtts_text_condition", "fa_luxtts_text_condition_device"):
        getattr(L, name).argtypes = [vp, i32, vp, vp, i64, i64, vp]
    for name in ("fa_luxtts_model_inputs", "fa_luxtts_model_inputs_device"):
        getattr(L, name).argtypes = [vp, i32, vp, vp, vp]
    for name in ("fa_luxtts_advance", "fa_luxtts_advance_device"):
        getattr(L, name).argtypes = [vp, i32, vp, vp, i64, i64]
    for name in ("fa_luxtts_vocoder_input", "fa_luxtts_vocoder_input_device"):
        getattr(L, name).argtypes = [vp, i32, vp, i32, vp]
    for name in ("fa_luxtts_finish", "fa_luxtts_finish_device"):
        getattr(L, name).argtypes = [vp, i32, vp, vp, i64, i64, vp, sz, vp, C.POINTER(i64)]
    L.fa_luxtts_close.argtypes = [vp, i32]
    L.fa_luxtts_request_state.argtypes = [vp, i32, LP, vp]
    for name in LUXTTS_SYMBOLS:
        if name != "fa_luxtts_destroy":
            getattr(L, name).restype = C.c_int
    L.fa_styletts2_plan.argtypes = [i32, C.POINTER(i32), C.POINTER(i32)]
    for name in ("fa_styletts2_sampler_inputs", "fa_styletts2_sampler_inputs_device"):
        getattr(L, name).argtypes = [i32, vp, vp, vp, i32, vp, vp, vp, vp]
    for name in ("fa_styletts2_style", "fa_styletts2_style_device"):
        getattr(L, name).argtypes = [i32, vp, vp, vp, vp, vp, vp]
    for name in ("fa_styletts2_align", "fa_styletts2_align_device"):
        getattr(L, name).argtypes = [i32, vp, vp, i32, i64, i64, vp, i32, i64, i64, vp, i32, i64, i64, i64, vp, vp, vp,
                                     vp, vp]
    for name in STYLETTS2_SYMBOLS:
        getattr(L, name).restype = C.c_int
    L.fa_offline_sortformer_plan.argtypes = [i32, i32, vp, vp, vp]
    for name in ("fa_offline_sortformer_model_inputs", "fa_offline_sortformer_model_inputs_device"):
        getattr(L, name).argtypes = [i32, i32, vp, vp, vp, i64, vp, vp]
    for name in ("fa_offline_sortformer_stitch", "fa_offline_sortformer_stitch_device"):
        getattr(L, name).argtypes = [i32, i32, vp, vp, vp, vp]
    for name in OFFLINE_SORTFORMER_SYMBOLS:
        getattr(L, name).restype = C.c_int
    _lib = L
    return L


def check(status: int, where: str) -> None:
    if status != 0:
        raise FluidAudioError(int(status), where, load().fa_last_error().decode("utf-8", "replace"))


def ptr(a):
    """Raw data pointer of a C-contiguous numpy array (None passes NULL)."""
    return None if a is None else a.ctypes.data


def device_count() -> int:
    return int(load().fa_device_count())


def set_device(ordinal: int) -> None:
    check(load().fa_set_device(ordinal), "fa_set_device")


def synchronize() -> None:
    check(load().fa_device_synchronize(), "fa_device_synchronize")


def kernel_launch_count() -> int:
    return int(load().fa_kernel_launch_count())


class PinnedArray:
    """numpy view over page-locked host memory from fa_host_alloc (so H2D/D2H copies run at link speed)."""

    def __init__(self, shape, dtype):
        self.shape = tuple(int(s) for s in np.atleast_1d(shape))
        self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = C.c_void_p()
        check(load().fa_host_alloc(max(nbytes, 1), C.byref(p)), "fa_host_alloc")
        self._p = p
        buf = (C.c_char * max(nbytes, 1)).from_address(p.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def free(self):
        if self._p is not None:
            self.array = None
            load().fa_host_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class DeviceBuffer:
    """Raw HBM allocation (fa_device_alloc) for the device-resident entry points."""

    def __init__(self, nbytes: int):
        p = C.c_void_p()
        check(load().fa_device_alloc(max(int(nbytes), 1), C.byref(p)), "fa_device_alloc")
        self.ptr = p
        self.nbytes = int(nbytes)

    def upload(self, a: np.ndarray):
        a = np.ascontiguousarray(a)
        check(load().fa_memcpy_h2d(self.ptr, a.ctypes.data, a.nbytes), "fa_memcpy_h2d")

    def download(self, shape, dtype) -> np.ndarray:
        out = np.empty(shape, dtype)
        check(load().fa_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes), "fa_memcpy_d2h")
        return out

    def free(self):
        if self.ptr is not None:
            load().fa_device_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
