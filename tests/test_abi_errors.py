"""Every failing C ABI call leaves fa_last_error() text that describes its own failure (CPU, and unchanged on the GPU).

Each status-returning entry point the headers declare is called once with arguments the library refuses in its own
argument checks, before any CUDA call: a null handle, a null required pointer, a negative count or an invalid config.
Before each call another call leaves a known text; the refused call must return the status pinned here and replace
that text with its own.  The source checks keep the one guard (fluidaudio_b200/csrc/c_abi.h) the only place that maps
exceptions to statuses, and every status-returning entry point a body that returns through it.
"""
import ctypes as C
import os
import re
import sys

import pytest

from fluidaudio_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from csrc_sources import ROOT, path, sources  # noqa: E402

N = None   # a null pointer
i32, i64, u64, sz, f32, f64 = C.c_int32, C.c_int64, C.c_uint64, C.c_size_t, C.c_float, C.c_double

# entry point -> (status the library returns, arguments it refuses before touching the device)
REFUSED = {
    "fa_host_alloc": (1, [sz(0), N]),
    "fa_device_alloc": (1, [sz(0), N]),
    "fa_memcpy_probe": (1, [N, sz(0), N, sz(0), i32(0), N]),
    "fa_timer_stop_ms": (1, [N]),
    "fa_mel_create": (1, [N, N]),
    "fa_mel_create_ex": (1, [N, N]),
    "fa_mel_cohere_features": (1, [N, N, sz(0), i64(-1), N, sz(0), N, N]),
    "fa_mel_styletts2_features": (1, [N, N, sz(0), N, sz(0), N]),
    "fa_mel_luxtts_features": (1, [N, N, sz(0), N, sz(0), N]),
    "fa_mel_get_window": (1, [N, N, sz(0)]),
    "fa_mel_get_filterbank": (1, [N, N, sz(0)]),
    "fa_mel_set_precision": (1, [N, i32(0)]),
    "fa_mel_set_pipeline_chunks": (1, [N, i32(1)]),
    "fa_mel_set_zero_copy_output": (1, [N, i32(0)]),
    "fa_mel_compute": (1, [N, N, sz(0), f32(0), i32(0), i64(-1), i32(0), N, sz(0), N, N]),
    "fa_mel_compute_device": (1, [N, N, sz(0), f32(0), i32(0), i64(-1), i32(0), N, sz(0), N, N]),
    "fa_mel_compute_batch": (1, [N, N, N, i32(0), N, i32(0), i32(0), N, N, N, N]),
    "fa_mel_compute_batch_device": (1, [N, N, N, i32(0), N, i32(0), i32(0), N, N, N, N]),
    "fa_mel_stream_open": (1, [N, N]),
    "fa_mel_stream_close": (1, [N, i32(0)]),
    "fa_mel_stream_push": (1, [N, i32(0), N, N, N, N, N, sz(0), N]),
    "fa_mel_stream_push_device": (1, [N, i32(0), N, N, N, N, N, sz(0), N]),
    "fa_mel_timer_start": (1, [N]),
    "fa_mel_timer_stop_ms": (1, [N, N]),
    "fa_mel_unified_features": (1, [N, N, sz(0), sz(0), N, sz(0), N, N]),
    "fa_mel_lseend_features": (1, [N, N, sz(0), N, N, N, sz(0), N]),
    "fa_mel_normalize_per_feature": (1, [N, i64(0), i32(0), i64(0)]),
    "fa_audio_resample": (1, [N, i64(-1), "format", N, i64(0), N]),
    "fa_audio_to_mel": (1, [N, N, i64(0), N, f32(0), i32(0), i32(0), N, sz(0), N, N, N]),
    "fa_linear_resample": (1, [N, i64(-1), i32(1), f64(16000), f64(16000), N, i64(0), N]),
    "fa_l2_normalize_rows": (1, [N, sz(1), sz(1), N]),
    "fa_ahc_cluster": (1, [N, sz(2), sz(1), f64(0.5), N]),
    "fa_dendrogram_cut": (1, [N, sz(2), f64(0.5), N]),
    "fa_vbx_refine": (1, [N, sz(0), sz(0), N, sz(0), N, i32(0), N, N, N, N, N, N]),
    "fa_compute_centroids": (1, [N, sz(0), sz(0), N, N, i32(0), N, N]),
    "fa_assign_embeddings": (1, [N, sz(1), sz(1), N, i32(0), N, N]),
    "fa_diarize_cluster": (1, [N, N, sz(0), sz(0), sz(0), N, N, N, N, N, i32(0), N]),
    "fa_diarize_cluster_chunks": (1, [N, N, sz(0), sz(0), sz(0), N, N, N, N, N, N, i32(0), N]),
    "fa_hungarian_solve": (1, [N, i32(-1), N]),
    "fa_max_score_assignment": (1, [N, i32(-1), i32(0), N]),
    "fa_constrained_assign": (1, [N, sz(1), i32(-1), N, N]),
    "fa_build_chunk_assignments": (1, [N, N, N, sz(0), i32(-1), i32(0), i32(0), N]),
    "fa_build_segments": (1, [N, i32(0), i32(0), i32(0), N, i32(0), N, i32(0), i32(0), N, N, N, N, N, i32(0), N]),
    "fa_build_speaker_database": (1, [N, i32(-1), N, i32(0), i32(0), N, N]),
    "fa_seg_window_count": (1, [i64(-1), N, N, N, N]),
    "fa_seg_windows": (1, [N, i64(-1), N, i32(0), i32(0), N, N]),
    "fa_seg_windows_device": (1, [N, i64(-1), N, i32(0), i32(0), N, N]),
    "fa_seg_decode": (1, [N, i32(-1), i32(0), i32(1), N, N, N, N, N]),
    "fa_seg_decode_device": (1, [N, i32(-1), i32(0), i32(1), N, N, N, N, N]),
    "fa_embedding_plan": (1, [N, i32(-1), i32(0), i32(0), N, i32(0), f64(0), i64(0), N, N] + [N] * 13),
    "fa_embedding_plan_device": (1, [N, i32(-1), i32(0), i32(0), N, i32(0), f64(0), i64(0), N, N] + [N] * 13),
    "fa_embed_windows": (1, [N, i64(-1), N, i32(0), N, i32(0), N, i32(1), N]),
    "fa_embed_windows_device": (1, [N, i64(-1), N, i32(0), N, i32(0), N, i32(1), N]),
    "fa_weight_resample": (1, [N, i64(-1), i32(1), i32(1), N]),
    "fa_kmeans_cluster": (1, [N, sz(1), sz(1), i32(1), i32(10), i32(1), u64(0), N, N, i32(0), N, N]),
    "fa_speaker_constraints_resolve": (1, [i64(0), i64(0), i64(0), i64(0), N, N]),
    "fa_export_shape": (1, [N, N, N, N]),
    "fa_export_read": (1, [N, sz(0), sz(0), sz(0)] + [N] * 9),
    "fa_export_write": (1, [N, sz(0), sz(0), sz(0)] + [N] * 9),
    "fa_diarize_cluster_batch": (1, [N, N, N, i32(0), sz(0), sz(0), N, N, N, N]),
    "fa_diarize_cluster_batch_chunks": (1, [N, N, N, i32(0), sz(0), sz(0), N, N, N, N, N]),
    "fa_sortformer_default_config": (1, [N, i32(0)]),
    "fa_sortformer_resolve_config": (1, [N, i32(0), N, N]),
    "fa_sortformer_step": (1, [N, i32(0), N, i32(0), i32(0), i32(0), i32(0), N]),
    "fa_sortformer_create": (1, [N, i32(0), N]),
    "fa_sortformer_open": (1, [N, N]),
    "fa_sortformer_close": (1, [N, i32(0)]),
    "fa_sortformer_update": (1, [N, i32(0), N, N, i32(0), N, i32(0), N, N, N, N, sz(0), N, sz(0), N, N]),
    "fa_sortformer_update_device": (1, [N, i32(0), N, N, i32(0), N, i32(0), N, N, N, N, sz(0), N, sz(0), N, N]),
    "fa_sortformer_model_inputs": (1, [N, i32(0), N, N, N, N, N]),
    "fa_sortformer_model_inputs_device": (1, [N, i32(0), N, N, N, N, N]),
    "fa_sortformer_session_state": (1, [N, i32(0), N, N, N, N, N, N]),
    "fa_diarizer_timeline_default_config": (1, [N, i32(0), i32(1), f32(0.1)]),
    "fa_diarizer_timeline_config_from_seconds": (1, [N, f32(0), f32(0), f32(0), f32(0)]),
    "fa_diarizer_timeline_segment_bound": (1, [i32(0), i32(0), N, N, N, N]),
    "fa_diarizer_timeline_create": (1, [N, i32(0), N]),
    "fa_diarizer_timeline_open": (1, [N, N]),
    "fa_diarizer_timeline_close": (1, [N, i32(0)]),
    "fa_diarizer_timeline_push": (1, [N, i32(0), N, N, N, N, N, N, sz(0), N, sz(0), N, N]),
    "fa_diarizer_timeline_push_device": (1, [N, i32(0), N, N, N, N, N, N, sz(0), N, sz(0), N, N]),
    "fa_diarizer_timeline_finalize": (1, [N, i32(0), N]),
    "fa_diarizer_timeline_reset": (1, [N, i32(0), N]),
    "fa_diarizer_timeline_clear_speaker": (1, [N, i32(0), i32(0)]),
    "fa_diarizer_timeline_session_state": (1, [N, i32(0), N, N, N, N]),
    "fastcluster_compute_centroid_linkage": (1, [N, sz(3), sz(2), N, sz(8)]),
}

# counting entry points -> (result type, arguments they refuse with -1)
REFUSED_COUNTS = {
    "fa_mel_frame_count": (i64, [N, i64(0), i32(0), i64(-1)]),
    "fa_mel_get_precision": (i32, [N]),
    "fa_mel_stream_frames": (i64, [N, i32(0), i64(0), i32(0)]),
    "fa_resample_output_count": (i64, [N, i64(0)]),
}

NO_ARGUMENT_FAILURE = {
    # text, counts and nothing to refuse
    "fa_version", "fa_last_error", "fa_device_count", "fa_kernel_launch_count", "fa_ahc_last_stage_ms",
    # void: defaults into a caller struct, NULL ignored
    "fa_mel_default_config", "fa_mel_ex_default_config", "fa_mel_preset_cohere", "fa_mel_preset_styletts2",
    "fa_mel_preset_luxtts", "fa_vbx_default_config", "fa_cluster_default_config", "fa_reconstruct_default_config",
    "fa_seg_default_config", "fa_embed_plan_default_config",
    "fa_mel_destroy", "fa_sortformer_destroy", "fa_diarizer_timeline_destroy",
    "fa_host_free", "fa_device_free",   # NULL is a no-op
    # every failure is the device's
    "fa_set_device", "fa_device_synchronize", "fa_timer_start", "fa_memcpy_h2d", "fa_memcpy_d2h",
}


FAMILY_HEADERS = ("fluidaudio_b200_ctc.h", "fluidaudio_b200_ctc_decode.h", "fluidaudio_b200_lseend.h",
                  "fluidaudio_b200_online_diar.h", "fluidaudio_b200_vad.h")   # each family's test_*_abi.py refuses its own


def _declared(headers=("fluidaudio_b200.h", "FastClusterWrapper.h")):
    names = set()
    for header in headers:
        text = open(os.path.join(ROOT, "include", header)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names |= set(re.findall(r"\b(fa_[a-z0-9_]+|fastcluster_compute_centroid_linkage)\s*\(", text))
    return names


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = C.CDLL(_lib.LIB_PATH)   # its own function objects: every argument below carries its C type
    L.fa_last_error.restype = C.c_char_p
    for name, (restype, _) in REFUSED_COUNTS.items():
        getattr(L, name).restype = restype
    return L


def _leave_sentinel(L):
    """a refused call that sets its own text"""
    fmt = _lib.AudioFormat(0.0, 16000.0, 1, 0, 0, 0)
    count = C.c_int64()
    assert L.fa_audio_resample(N, i64(10), C.byref(fmt), N, i64(0), C.byref(count)) == 1
    text = L.fa_last_error()
    assert text.startswith(b"audio format:")
    return text


def test_every_declared_entry_point_is_covered():
    covered = set(REFUSED) | set(REFUSED_COUNTS)
    assert not covered & NO_ARGUMENT_FAILURE
    assert covered | NO_ARGUMENT_FAILURE == _declared()


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_a_refused_call_reports_its_own_failure(lib, name):
    status, args = REFUSED[name]
    fmt = _lib.AudioFormat(16000.0, 16000.0, 1, 0, 0, 0)   # a valid format, for the calls that take one
    args = [C.byref(fmt) if a == "format" else a for a in args]
    sentinel = _leave_sentinel(lib)
    assert getattr(lib, name)(*args) == status
    text = lib.fa_last_error()
    assert text and text != sentinel, f"{name} left {text!r}"


@pytest.mark.parametrize("name", sorted(REFUSED_COUNTS))
def test_a_refused_count_reports_its_own_failure(lib, name):
    sentinel = _leave_sentinel(lib)
    assert getattr(lib, name)(*REFUSED_COUNTS[name][1]) == -1
    text = lib.fa_last_error()
    assert text and text != sentinel, f"{name} left {text!r}"


def test_a_successful_call_leaves_the_text(lib):
    sentinel = _leave_sentinel(lib)
    lo, hi = C.c_int64(), C.c_int64()
    assert lib.fa_speaker_constraints_resolve(i64(10), i64(-1), i64(-1), i64(-1), C.byref(lo), C.byref(hi)) == 0
    assert lib.fa_last_error() == sentinel


def _code(name):
    """source without comments, string and character literals"""
    with open(path(name), encoding="utf-8") as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    return re.sub(r'"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', '""', text)


def test_only_the_guard_maps_exceptions():
    catches = {}
    for name in sources():
        for m in re.finditer(r"\bcatch\s*\(\s*(?:const\s+)?std::(bad_alloc|exception)\b", _code(name)):
            catches.setdefault(m.group(1), []).append(name)
    assert catches == {"bad_alloc": ["c_abi.h"], "exception": ["c_abi.h"]}


def test_every_status_entry_point_returns_through_the_guard():
    guarded, offenders = set(), []
    for name in sources():
        code = _code(name)
        for m in re.finditer(r"\bFA_API\s+(fa_status|fastcluster_wrapper_status)\s+(\w+)\s*\(", code):
            i = code.index("{", m.end())
            depth, j = 1, i + 1
            statements = 0
            while depth:
                c = code[j]
                depth += {"{": 1, "(": 1, "[": 1, "}": -1, ")": -1, "]": -1}.get(c, 0)
                statements += c == ";" and depth == 1
                j += 1
            body = " ".join(code[i + 1:j - 1].split())
            if statements == 1 and re.match(r"return (to_fc\()?(fa::)?guard\(__func__, ", body):
                guarded.add(m.group(2))
            else:
                offenders.append(f"{name}: {m.group(2)}")
    assert not offenders, f"entry points that return other than through guard(): {offenders}"
    declared_status = {n for n in _declared() if n in REFUSED or n in
                       {"fa_set_device", "fa_device_synchronize", "fa_timer_start", "fa_memcpy_h2d", "fa_memcpy_d2h",
                        "fa_host_free", "fa_device_free"}}
    assert guarded - _declared(FAMILY_HEADERS) == declared_status
