/* Plain-C consumer of the drop-in boundary: proves that the headers under include/ are valid C (not only C++) and that the shared
 * library links and runs from C without a GPU for everything that is host-only.  Built and run by
 * tests/test_host_logic.py::test_headers_are_plain_c_and_link. */
#include "FastClusterWrapper.h"
#include "fluidaudio_b200.h"

#include <stdio.h>
#include <string.h>

int main(void) {
    const char *v = fa_version();
    if (!v || !strstr(v, "sm_90a")) return 1;

    /* the reference's argument contract needs no device (FastClusterWrapper.cpp:203-216) */
    double x[4] = {1.0, 0.0, 0.0, 1.0}, z[4];
    if (fastcluster_compute_centroid_linkage(NULL, 2, 2, z, 4) != FASTCLUSTER_WRAPPER_INVALID_ARGUMENT) return 2;
    if (fastcluster_compute_centroid_linkage(x, 0, 2, z, 4) != FASTCLUSTER_WRAPPER_SUCCESS) return 3;
    if (fastcluster_compute_centroid_linkage(x, 2, 2, z, 3) != FASTCLUSTER_WRAPPER_OUTPUT_TOO_SMALL) return 4;

    /* host-only entry points */
    int64_t lo = 0, hi = 0;
    if (fa_speaker_constraints_resolve(5, FA_NO_VALUE, 2, 20, &lo, &hi) != FA_STATUS_OK || lo != 2 || hi != 5) return 5;
    int64_t cost[9] = {4, 1, 3, 2, 0, 5, 3, 2, 2};
    int32_t assign[3] = {-1, -1, -1};
    if (fa_hungarian_solve(cost, 3, assign) != FA_STATUS_OK) return 6;
    if (assign[0] != 1 || assign[1] != 0 || assign[2] != 2) return 7;   /* 1 + 2 + 2 = 5 is the optimum */

    fa_cluster_config cfg;
    fa_cluster_default_config(&cfg);
    if (cfg.threshold != 0.6 || cfg.num_speakers != FA_NO_VALUE) return 8;
    fa_mel_config mc;
    fa_mel_default_config(&mc);
    if (mc.n_fft != 512 || mc.hop_length != 160) return 9;

    /* timeline reconstruction: one chunk, four frames of 0.5 s, local speaker 0 -> cluster 1 */
    {
        fa_reconstruct_config rc;
        fa_reconstruct_default_config(&rc);
        rc.frame_duration = 0.5;
        rc.min_segment_duration = 0.0;
        const float weights[8] = {0.9f, 0.0f, 0.9f, 0.0f, 0.9f, 0.0f, 0.9f, 0.0f};
        const int32_t hard[2] = {1, -2};
        const double offsets[1] = {0.0};
        int32_t cl[4], count = 0;
        float st[4], en[4], q[4];
        if (fa_build_segments(weights, 1, 4, 2, offsets, 1, hard, 1, 2, &rc, cl, st, en, q, 4, &count) != FA_STATUS_OK) return 10;
        if (count != 1 || cl[0] != 1 || st[0] != 0.0f || en[0] != 2.0f) return 11;
    }

    {   /* converter stage: sizing and argument checks are host-side (AudioConverter.swift:417-418: Int(n / ratio)) */
        fa_audio_format af;
        int64_t n_out = -1;
        af.in_rate = 44100.0;
        af.out_rate = 16000.0;
        af.channels = 2;
        af.format = FA_PCM_I16;
        af.interleaved = 1;
        af.algorithm = FA_RESAMPLE_AUTO;
        if (fa_resample_output_count(&af, 44100) != 16000) return 12;
        if (fa_audio_resample(NULL, 44100, &af, NULL, 0, &n_out) != FA_STATUS_OK || n_out != 16000) return 13;
        af.channels = 0;
        if (fa_audio_resample(NULL, 44100, &af, NULL, 0, &n_out) != FA_STATUS_INVALID_ARGUMENT) return 14;
    }
    printf("abi ok: %s, devices visible: %d\n", v, fa_device_count());
    return 0;
}
