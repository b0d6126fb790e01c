// Host-buffer pipelines of the log-mel plan: host samples in, host rows out, with the copies of one unit overlapping the
// kernels of the next (MelPlan::compute_host: one clip, any AudioFormat, through the converter stage; compute_batch_host:
// a batch of float32 clips in groups).  The launches themselves are MelPlan::launch (mel_kernels.cu).  Also the plan's
// event timer on its compute stream (fa_mel_timer_*).
#include "mel_core.cuh"
#include "mel_plan.h"

#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace fa {
namespace mel {

// A pinned (page-locked, mapped) host buffer has a device alias under UVA: the kernel can then store its output rows
// straight into host memory (coalesced 16-byte stores become posted PCIe writes), which removes the D2H copy stage and its
// cross-stream hand-offs from the pipeline.  Pageable memory returns nullptr and takes the staged copy.
static float *device_alias_if_pinned(float *host) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, host) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return (a.type == cudaMemoryTypeHost && a.devicePointer) ? static_cast<float *>(a.devicePointer) : nullptr;
}

// FA_MEL_TRACE_PIPELINE=1: device timestamps (timing events) at the end of every unit's H2D, kernels and D2H of the
// host-buffer pipeline (MelPlan::compute_host), printed to stderr after the call.  Off: no events, no cost.
struct PipelineTrace {
    bool on = false;
    Event t0;
    std::vector<Event> ev;
    std::vector<int> tag;   // unit * 4 + stage (0 H2D done, 1 kernels done, 2 D2H done)
    PipelineTrace() {
        static const bool want = [] { const char *e = std::getenv("FA_MEL_TRACE_PIPELINE"); return e && *e && *e != '0'; }();
        on = want;
    }
    void start(cudaStream_t s) {
        if (!on) return;
        t0.create();
        cudaEventRecord(t0, s);
    }
    void mark(cudaStream_t s, int unit, int stage) {
        if (!on) return;
        ev.emplace_back();
        ev.back().create();
        cudaEventRecord(ev.back(), s);
        tag.push_back(unit * 4 + stage);
    }
    void dump(const char *what) {
        if (!on) return;
        static const char *names[3] = {"h2d", "kern", "d2h"};
        std::fprintf(stderr, "[pipeline %s]", what);
        for (size_t i = 0; i < ev.size(); ++i) {
            float ms = 0.0f;
            cudaEventElapsedTime(&ms, t0, ev[i]);
            std::fprintf(stderr, " u%d.%s=%.3f", tag[i] / 4, names[tag[i] & 3], ms);
        }
        std::fprintf(stderr, "\n");
    }
};

// Frame ranges of the pipeline's units.  The pipeline's fixed cost is its ramp: nothing can be computed before the first
// unit's samples have landed, and the last unit's kernel + D2H run after the last byte of input.  So the units at both ends
// are small (1 : 2 : 4 ... 4 : 2 : 1) and the ones in between large enough to amortise the per-transfer cost.  Bounds are
// multiples of the tile height; no unit is shorter than min_unit frames (fewer units otherwise).
static std::vector<long long> unit_bounds(long long T, long long max_units, long long min_unit) {
    std::vector<long long> b{0};
    long long K = std::max<long long>(1, std::min(max_units, T / std::max<long long>(1, min_unit)));
    auto weight = [&](long long c, long long k) -> long long {
        if (k < 6) return 4;
        const long long e = std::min(c, k - 1 - c);
        return e == 0 ? 1 : (e == 1 ? 2 : 4);
    };
    for (; K > 1; --K) {   // the smallest unit must still hold min_unit frames
        long long sum = 0;
        for (long long c = 0; c < K; ++c) sum += weight(c, K);
        if (T * weight(0, K) / sum >= min_unit) break;
    }
    long long sum = 0, acc = 0;
    for (long long c = 0; c < K; ++c) sum += weight(c, K);
    for (long long c = 0; c + 1 < K; ++c) {
        acc += weight(c, K);
        const long long e = std::min(T, ceil_to((long long)((double)T * (double)acc / (double)sum), kTileFrames));
        if (e > b.back() && e < T) b.push_back(e);
    }
    b.push_back(T);
    return b;
}

int MelPlan::ensure_resampler(double in_rate, double out_rate) {
    if (in_rate == out_rate || (in_rate == rs_in && out_rate == rs_out && d_rs_tab.data())) return FA_OK;
    resample::Design d;
    int st = resample::make_design(in_rate, out_rate, d);
    if (st != FA_OK) return st;
    rs_in = rs_out = 0.0;   // the table is being replaced
    st = d_rs_tab.grow(d.table.size() * sizeof(float));
    if (st != FA_OK) return st;
    // on the compute stream, which runs the conversion; complete before `d` is moved
    FA_CUDA_TRY(cudaMemcpyAsync(d_rs_tab.data(), d.table.data(), d.table.size() * sizeof(float), cudaMemcpyHostToDevice,
                                streams[1]));
    FA_CUDA_TRY(cudaStreamSynchronize(streams[1]));
    rs_design = std::move(d);
    rs_in = in_rate;
    rs_out = out_rate;
    return FA_OK;
}

// Host buffers in, host buffers out: AudioConverter.resample + computeFlatTransposed as one device pipeline.  A long
// clip is cut into units.  The PCM is copied in chunks; as soon as a chunk has landed the compute stream converts the
// samples it completes (mixdown + polyphase / linear, see resample_kernels.cu) into the float buffer the mel kernel
// reads, runs the frames those samples complete, and the D2H stream returns their rows — H2D of unit c+1, kernels of
// unit c and D2H of unit c-1 overlap.  Identity input (mono float32 at the model rate) is copied straight into the float
// buffer and needs no conversion kernel.
int MelPlan::compute_host(const void *pcm, long long frames, const resample::AudioFormat &f, float last, int mode,
                          long long expected, int layout, float *out, long long out_len, long long *mel_length,
                          long long *num_frames, long long *resampled) {
    const long long n = resample::output_count(frames, f.in_rate, f.out_rate);
    if (resampled) *resampled = n;
    long long T, Tp;
    int st = clip_shape(*this, n, mode, expected, out_len, T, Tp, mel_length, num_frames);
    if (st != FA_OK) return st;
    if (T == 0) {
        if (Tp) std::fill(out, out + cfg.n_mels, 0.0f);   // padValue
        return FA_OK;
    }
    const bool identity = resample::is_identity(f);
    const long long need = Tp * cfg.n_mels;
    st = ensure_resampler(f.in_rate, f.out_rate);
    if (st != FA_OK) return st;
    const size_t bps = f.format == resample::kPcmI16 ? 2 : 4;
    const size_t pcm_bytes = (size_t)frames * f.channels * bps;
    float *d_f32, *d_rows;   // kernel input, staged output
    char *d_pcm = nullptr;   // the raw PCM of converted input
    st = carve_arena(staging, [&](Carver &c) {
        d_f32 = c.take<float>((size_t)n + 8);
        d_rows = c.take<float>((size_t)need);
        if (!identity) d_pcm = c.take<char>(pcm_bytes + 16);
    });
    if (st != FA_OK) return st;
    char *const d_in = identity ? reinterpret_cast<char *>(d_f32) : d_pcm;   // where the input lands
    // Units: pipeline_chunks for identity input; converted input keeps ~10 MB of PCM per unit (the copy engines' fixed
    // cost per transfer and the host's enqueue rate make finer units slower there: int16 hour 3.08 ms at 8-12 units,
    // 3.44 at 24, 3.61 at 96).
    const long long max_units =
        identity ? pipeline_chunks : std::min<long long>(pipeline_chunks, (long long)(pcm_bytes / (10u << 20)) + 1);
    const std::vector<long long> bounds = unit_bounds(T, max_units, 4096);
    const int chunks = (int)bounds.size() - 1;
    // A single unit is the streaming callers' shape (a few thousand samples, SortformerDiarizer.swift:857-905): nothing
    // to overlap, so one stream, no events, the unit descriptor passed in the kernel parameters, one synchronisation.
    const bool single = chunks == 1;
    float *out_alias = (zero_copy_out && layout == FA_MEL_TIME_MAJOR && !single) ? device_alias_if_pinned(out) : nullptr;
    float *k_out = out_alias ? out_alias : d_rows;   // where the kernel writes
    if (out_alias && Tp > T) std::memset(out + T * cfg.n_mels, 0, (size_t)(Tp - T) * cfg.n_mels * sizeof(float));
    st = units.reserve(unit_bytes(chunks));
    if (st != FA_OK) return st;
    st = ensure_events(2 * (size_t)chunks);
    if (st != FA_OK) return st;
    cudaStream_t s_k = streams[1], s_in = single ? s_k : streams[0], s_out = single ? s_k : streams[2];
    MelUnit *h_units = units.host.data();
    for (int c = 0; c < chunks; ++c) h_units[c] = MelUnit{0, n, 0, Tp, bounds[c], bounds[c + 1] - bounds[c], last, 0};
    if (!single) {
        st = units.upload(chunks * sizeof(MelUnit), s_k);
        if (st != FA_OK) return st;
    }
    const long long pad = mode == FA_MEL_PAD_CENTER ? cfg.n_fft / 2 : 0;
    const resample::Design &D = rs_design;
    const bool linear = f.in_rate != f.out_rate && resample::resolve_algorithm(f) == resample::kAlgoLinear;
    long long in_copied = 0, converted = 0;
    PipelineTrace trace;
    trace.start(s_in);
    for (int c = 0; c < chunks; ++c) {
        const bool tail = c == chunks - 1;
        // model-rate samples needed so far, and the input frames those samples depend on
        long long s_end = tail ? n : std::min(n, (bounds[c + 1] - 1) * cfg.hop_length + cfg.n_fft - pad);
        // Reflected .center frames read the clip's end only when they cross it (then s_end = n already), and a frame
        // crossing the start reads up to x[pad] (reflect_index): every unit's range must hold that sample.
        if (mode == FA_MEL_PAD_CENTER && cfg.reflect()) s_end = std::min(n, std::max(s_end, pad + 1));
        long long in_need = frames;
        if (!tail) {
            if (f.in_rate == f.out_rate) in_need = s_end;
            else if (linear) in_need = (long long)((double)(s_end + 1) * (f.in_rate / f.out_rate)) + 4;
            else in_need = ((s_end + 2) * D.M) / D.L + D.half + 3;
            in_need = std::min(frames, std::max(in_need, in_copied));
        }
        if (in_need > in_copied) {
            const char *src = static_cast<const char *>(pcm);
            if (f.interleaved || f.channels == 1) {
                const size_t a = (size_t)in_copied * f.channels * bps, b = (size_t)in_need * f.channels * bps;
                FA_CUDA_TRY(cudaMemcpyAsync(d_in + a, src + a, b - a, cudaMemcpyHostToDevice, s_in));
            } else {
                for (int ch = 0; ch < f.channels; ++ch) {
                    const size_t a = ((size_t)ch * frames + in_copied) * bps, b = ((size_t)ch * frames + in_need) * bps;
                    FA_CUDA_TRY(cudaMemcpyAsync(d_in + a, src + a, b - a, cudaMemcpyHostToDevice, s_in));
                }
            }
            in_copied = in_need;
        }
        // zero the pad rows after the first input copy: a copy from pageable memory first waits for its stream's queue
        if (c == 0 && Tp > T && !out_alias) FA_CUDA_TRY(cudaMemsetAsync(d_rows, 0, need * sizeof(float), s_k));
        if (!single) {
            FA_CUDA_TRY(cudaEventRecord(events[2 * c], s_in));
            FA_CUDA_TRY(cudaStreamWaitEvent(s_k, events[2 * c], 0));
        }
        trace.mark(s_in, c, 0);
        if (!identity) {
            const long long ready = resample::outputs_ready(f, D, frames, in_copied, n);
            if (ready < s_end) {
                fa::set_error("internal: resampler window accounting (%lld < %lld)", ready, s_end);
                return FA_RUNTIME_ERROR;
            }
            st = resample::launch_convert(d_pcm, frames, f, D, d_rs_tab.data(), d_f32, converted, s_end, s_k);
            if (st != FA_OK) return st;
            converted = std::max(converted, s_end);
        }
        st = launch(units.device.data() + c, h_units + c, 1, single, d_f32, k_out, mode, layout, s_k);
        if (st != FA_OK) return st;
        trace.mark(s_k, c, 1);
        if (out_alias) continue;   // the kernel stored its rows in the caller's pinned buffer: no D2H stage
        if (!single) {
            FA_CUDA_TRY(cudaEventRecord(events[2 * c + 1], s_k));
            FA_CUDA_TRY(cudaStreamWaitEvent(s_out, events[2 * c + 1], 0));
        }
        const long long fb = bounds[c], rows = (tail ? Tp : bounds[c + 1]) - fb;   // the last unit also returns the pad rows
        if (layout == FA_MEL_TIME_MAJOR || single) {   // a single unit returns the whole buffer in either layout
            FA_CUDA_TRY(cudaMemcpyAsync(out + fb * cfg.n_mels, d_rows + fb * cfg.n_mels, rows * cfg.n_mels * sizeof(float),
                                        cudaMemcpyDeviceToHost, s_out));
        } else {
            FA_CUDA_TRY(cudaMemcpy2DAsync(out + fb, Tp * sizeof(float), d_rows + fb, Tp * sizeof(float),
                                          rows * sizeof(float), cfg.n_mels, cudaMemcpyDeviceToHost, s_out));
        }
        trace.mark(s_out, c, 2);
    }
    FA_CUDA_TRY(cudaStreamSynchronize(s_out));
    if (!single) FA_CUDA_TRY(cudaStreamSynchronize(s_k));
    trace.dump(identity ? "f32" : "pcm");
    return FA_OK;
}

// Batch of clips, host buffers: clips are grouped so that copies and kernels of successive groups overlap.
int MelPlan::compute_batch_host(const float *audio, const int64_t *offsets, int count, const float *last, int mode,
                                int layout, float *out, const int64_t *out_offsets, int64_t *mel_lengths,
                                int64_t *num_frames) {
    if (count <= 0) return FA_OK;
    // device-side packing: clip i starts at a 4-float aligned offset so that every tile can use the TMA path
    // When every clip already starts at a multiple of four floats in the caller's buffer, the device copy keeps the
    // caller's layout and a whole group of clips travels in ONE transfer (a bulk copy may read up to three floats past a
    // clip's end: the neighbour's samples or the pad below, never used: the kernel masks by the clip length).  512 clips
    // cost 1 024 cudaMemcpyAsync calls otherwise: ~4 ms of host enqueue time on a 25 ms batch.
    bool same_layout = true;
    for (int i = 0; i < count; ++i) same_layout = same_layout && ((offsets[i] - offsets[0]) & 3) == 0 && offsets[i + 1] >= offsets[i];
    std::vector<long long> doff(count + 1), dout(count + 1);
    long long a = 0, o = 0;
    std::vector<long long> Ts(count), Tps(count);
    for (int i = 0; i < count; ++i) {
        const long long n = offsets[i + 1] - offsets[i];
        doff[i] = same_layout ? offsets[i] - offsets[0] : a;
        a = same_layout ? ceil_to(offsets[i + 1] - offsets[0], 4) + 4 : a + ceil_to(n, 4) + 4;
        dout[i] = o;
        clip_shape(*this, n, mode, -1, kUnchecked, Ts[i], Tps[i], nullptr, nullptr);
        if (mel_lengths) mel_lengths[i] = Ts[i];
        if (num_frames) num_frames[i] = Tps[i];
        o += std::max<long long>(Tps[i], 1) * cfg.n_mels;   // an empty clip returns one zero row, in every mode
    }
    doff[count] = a;
    dout[count] = o;
    float *d_f32, *d_rows;
    int st = carve_arena(staging, [&](Carver &c) {
        d_f32 = c.take<float>((size_t)a + 8);
        d_rows = c.take<float>((size_t)o);
    });
    if (st != FA_OK) return st;
    st = units.reserve(unit_bytes(count));
    if (st != FA_OK) return st;
    const int groups = std::min(count, 32);   // one H2D, one launch, one D2H per group: the last group's kernel + D2H is the pipeline's tail
    st = ensure_events(2 * (size_t)groups);
    if (st != FA_OK) return st;
    cudaStream_t s_in = streams[0], s_k = streams[1], s_out = streams[2];
    // all unit descriptors first (one small copy), then per group: H2D, kernel, D2H
    MelUnit *h_units = units.host.data();
    std::vector<int> g_first(groups + 1);
    int used = 0;
    for (int g = 0; g < groups; ++g) {
        const int c0 = (int)((long long)count * g / groups), c1 = (int)((long long)count * (g + 1) / groups);
        g_first[g] = used;
        for (int i = c0; i < c1; ++i)
            if (Ts[i]) h_units[used++] = MelUnit{doff[i], offsets[i + 1] - offsets[i], dout[i], Tps[i], 0, Ts[i], last ? last[i] : 0.0f, 0};
        number_tiles(h_units + g_first[g], used - g_first[g]);
    }
    g_first[groups] = used;
    if (used) {
        st = units.upload(used * sizeof(MelUnit), s_k);
        if (st != FA_OK) return st;
    }
    FA_CUDA_TRY(cudaMemsetAsync(d_rows, 0, (size_t)o * sizeof(float), s_k));
    for (int g = 0; g < groups; ++g) {
        const int c0 = (int)((long long)count * g / groups), c1 = (int)((long long)count * (g + 1) / groups);
        if (same_layout) {
            const long long n = offsets[c1] - offsets[c0];
            if (n > 0)
                FA_CUDA_TRY(cudaMemcpyAsync(d_f32 + doff[c0], audio + offsets[c0], n * sizeof(float), cudaMemcpyHostToDevice, s_in));
        } else {
            for (int i = c0; i < c1; ++i) {
                const long long n = offsets[i + 1] - offsets[i];
                if (n > 0)
                    FA_CUDA_TRY(cudaMemcpyAsync(d_f32 + doff[i], audio + offsets[i], n * sizeof(float), cudaMemcpyHostToDevice, s_in));
            }
        }
        FA_CUDA_TRY(cudaEventRecord(events[2 * g], s_in));
        FA_CUDA_TRY(cudaStreamWaitEvent(s_k, events[2 * g], 0));
        st = launch(units.device.data() + g_first[g], h_units + g_first[g], g_first[g + 1] - g_first[g], false, d_f32, d_rows,
                    mode, layout, s_k);
        if (st != FA_OK) return st;
        FA_CUDA_TRY(cudaEventRecord(events[2 * g + 1], s_k));
        FA_CUDA_TRY(cudaStreamWaitEvent(s_out, events[2 * g + 1], 0));
        bool out_contiguous = c1 > c0;   // the caller's output offsets follow the packed device layout: one transfer
        for (int i = c0; i < c1 && out_contiguous; ++i) out_contiguous = out_offsets[i] - out_offsets[c0] == dout[i] - dout[c0];
        if (out_contiguous) {
            FA_CUDA_TRY(cudaMemcpyAsync(out + out_offsets[c0], d_rows + dout[c0], (dout[c1] - dout[c0]) * sizeof(float),
                                        cudaMemcpyDeviceToHost, s_out));
        } else {
            for (int i = c0; i < c1; ++i) {
                const long long len = dout[i + 1] - dout[i];
                FA_CUDA_TRY(cudaMemcpyAsync(out + out_offsets[i], d_rows + dout[i], len * sizeof(float), cudaMemcpyDeviceToHost, s_out));
            }
        }
    }
    FA_CUDA_TRY(cudaStreamSynchronize(s_out));
    FA_CUDA_TRY(cudaStreamSynchronize(s_k));
    return FA_OK;
}

int MelPlan::timer_start() {
    if (!timer[0]) {
        const int st = create_timer(timer);
        if (st != FA_OK) return st;
    }
    FA_CUDA_TRY(cudaStreamSynchronize(streams[1]));
    FA_CUDA_TRY(cudaEventRecord(timer[0], streams[1]));
    return FA_OK;
}

int MelPlan::timer_stop_ms(float *elapsed_ms) {
    if (!timer[0]) return FA_INVALID_ARGUMENT;
    FA_CUDA_TRY(cudaEventRecord(timer[1], streams[1]));
    FA_CUDA_TRY(cudaEventSynchronize(timer[1]));
    FA_CUDA_TRY(cudaEventElapsedTime(elapsed_ms, timer[0], timer[1]));
    return FA_OK;
}

} // namespace mel
} // namespace fa
