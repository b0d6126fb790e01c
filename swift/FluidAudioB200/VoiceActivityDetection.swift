// Voice activity detection (Sources/FluidAudio/VAD/) on the GPU (fa_vad_*, fa_fsmn_vad_decide): Silero live sessions
// as model_inputs / advance around the app's model, segmentSpeech for many clips, and the FSMN-VAD decision for many
// clips.  The CoreML models stay in the app.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func vadCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

private func offsets(_ counts: [Int]) -> [Int64] {
    var off: [Int64] = [0]
    for n in counts { off.append(off.last! + Int64(n)) }
    return off
}

/// VadConfig.defaultThreshold with VadSegmentationConfig's fields, as fa_vad_config.
public func makeVadConfig(defaultThreshold: Float = 0.85, minSpeechDuration: Double = 0.15,
                          minSilenceDuration: Double = 0.75, maxSpeechDuration: Double = 14.0,
                          speechPadding: Double = 0.1, silenceThresholdForSplit: Float = 0.3,
                          negativeThreshold: Float? = nil, negativeThresholdOffset: Float = 0.15,
                          minSilenceAtMaxSpeech: Double = 0.098,
                          useMaxPossibleSilenceAtMaxSpeech: Bool = true) -> fa_vad_config {
    fa_vad_config(default_threshold: defaultThreshold, min_speech_duration: minSpeechDuration,
                  min_silence_duration: minSilenceDuration, max_speech_duration: maxSpeechDuration,
                  speech_padding: speechPadding, silence_threshold_for_split: silenceThresholdForSplit,
                  has_negative_threshold: negativeThreshold == nil ? 0 : 1,
                  negative_threshold: negativeThreshold ?? 0, negative_threshold_offset: negativeThresholdOffset,
                  min_silence_at_max_speech: minSilenceAtMaxSpeech,
                  use_max_possible_silence_at_max_speech: useMaxPossibleSilenceAtMaxSpeech ? 1 : 0)
}

/// Silero VAD live sessions in HBM (fa_vad_stream).  A step is modelInputs, the app's model, then advance.
public final class SileroVadStreams {
    let handle: OpaquePointer

    public init() throws {
        var h: OpaquePointer?
        try vadCheck(fa_vad_stream_create(&h), "fa_vad_stream_create")
        handle = h!
    }

    deinit { fa_vad_stream_destroy(handle) }

    public func open() throws -> Int32 {
        var id: Int32 = 0
        try vadCheck(fa_vad_stream_open(handle, &id), "fa_vad_stream_open")
        return id
    }

    public func close(_ session: Int32) throws {
        try vadCheck(fa_vad_stream_close(handle, session), "fa_vad_stream_close")
    }

    /// (audio_input [n x 4160], hidden [n x 128], cell [n x 128]) for chunks[i] sent to sessions[i].
    public func modelInputs(sessions: [Int32], chunks: [[Float]]) throws -> ([Float], [Float], [Float]) {
        let audio = chunks.flatMap { $0 }
        let off = offsets(chunks.map { $0.count })
        var input = [Float](repeating: 0, count: sessions.count * Int(FA_VAD_MODEL_INPUT))
        var hidden = [Float](repeating: 0, count: sessions.count * Int(FA_VAD_STATE))
        var cell = hidden
        try vadCheck(fa_vad_stream_model_inputs(handle, Int32(sessions.count), sessions, audio, off, &input, &hidden,
                                                &cell), "fa_vad_stream_model_inputs")
        return (input, hidden, cell)
    }

    /// Commits the staged chunks; per session the event (kind 0 none, 1 start, 2 end) and its sample index.
    public func advance(sessions: [Int32], probability: [Float], newHidden: [Float], newCell: [Float],
                        config: fa_vad_config) throws -> [(kind: Int, sample: Int)] {
        var cfg = config
        var events = [Int64](repeating: 0, count: 2 * sessions.count)
        try vadCheck(fa_vad_stream_advance(handle, Int32(sessions.count), sessions, probability, newHidden, newCell,
                                           &cfg, &events), "fa_vad_stream_advance")
        return (0..<sessions.count).map { (Int(events[2 * $0]), Int(events[2 * $0 + 1])) }
    }
}

/// segmentSpeech(from:totalSamples:config:) for many clips: per clip, its (startTime, endTime) in seconds.
public func segmentSpeech(probabilities: [[Float]], totalSamples: [Int], config: fa_vad_config) throws
    -> [[(startTime: Double, endTime: Double)]] {
    let flat = probabilities.flatMap { $0 }
    let off = offsets(probabilities.map { $0.count })
    let totals = totalSamples.map { Int64($0) }
    var cfg = config
    var counts = [Int64](repeating: 0, count: probabilities.count)
    var segments = [Int64](repeating: 0, count: 2 * max(1, flat.count))
    var total: Int64 = 0
    try vadCheck(fa_vad_segment(flat, off, Int32(probabilities.count), totals, &cfg, &counts, &segments,
                                flat.count, &total), "fa_vad_segment")
    var out: [[(startTime: Double, endTime: Double)]] = []
    var at = 0
    for n in counts {
        out.append((0..<Int(n)).map { k in
            (Double(segments[2 * (at + k)]) / 16000.0, Double(segments[2 * (at + k) + 1]) / 16000.0)
        })
        at += Int(n)
    }
    return out
}

/// FsmnVadManager.decide(silence:) for many clips: per clip, its (startMs, endMs).
public func fsmnVadDecide(silence: [[Float]]) throws -> [[(startMs: Int, endMs: Int)]] {
    let flat = silence.flatMap { $0 }
    let off = offsets(silence.map { $0.count })
    var counts = [Int64](repeating: 0, count: silence.count)
    var segments = [Int64](repeating: 0, count: 2 * max(1, flat.count))
    var total: Int64 = 0
    try vadCheck(fa_fsmn_vad_decide(flat, off, Int32(silence.count), &counts, &segments, flat.count, &total),
                 "fa_fsmn_vad_decide")
    var out: [[(startMs: Int, endMs: Int)]] = []
    var at = 0
    for n in counts {
        out.append((0..<Int(n)).map { k in (Int(segments[2 * (at + k)]), Int(segments[2 * (at + k) + 1])) })
        at += Int(n)
    }
    return out
}
