// LuxTTS synthesis (Sources/FluidAudio/TTS/LuxTts/LuxTtsSynthesizer.swift) on the GPU (fa_luxtts_*): the host work
// between the text encoder, the FmDecoder and the vocoder for many requests per call.  The CoreML models stay in the
// app.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func luxCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

/// fa_luxtts_plan: the request geometry, or the reason code synthesize's guards refuse it with.
public func luxTtsPlan(promptSamples: Int, promptTokenCount: Int, textTokenCount: Int,
                       speed: Float) throws -> fa_luxtts_plan_info {
    var p = fa_luxtts_plan_info()
    try luxCheck(fa_luxtts_plan(Int64(promptSamples), Int32(promptTokenCount), Int32(textTokenCount), speed, &p),
                 "fa_luxtts_plan")
    return p
}

/// Live LuxTTS requests in HBM (fa_luxtts).  begin, textCondition, four x (modelInputs, FmDecoder, advance),
/// vocoderInput, vocoder, finish.
public final class LuxTtsRequests {
    let handle: OpaquePointer

    public init() throws {
        var h: OpaquePointer?
        try luxCheck(fa_luxtts_create(&h), "fa_luxtts_create")
        handle = h!
    }

    deinit { fa_luxtts_destroy(handle) }

    /// Opens one request per prompt; on a refusal `reasons` holds every request's code and nothing is opened.
    public func begin(prompts: [[Float]], promptTokenCounts: [Int32], textTokenCounts: [Int32], speeds: [Float],
                      seeds: [UInt64], reasons: inout [Int32], speechCondition: inout [Float],
                      paddingMask: inout [Float]) throws -> (ids: [Int32], plans: [fa_luxtts_plan_info]) {
        let n = prompts.count
        var off: [Int64] = [0]
        for p in prompts { off.append(off.last! + Int64(p.count)) }
        let audio = prompts.flatMap { $0 }
        var ids = [Int32](repeating: 0, count: n)
        var plans = [fa_luxtts_plan_info](repeating: fa_luxtts_plan_info(), count: n)
        reasons = [Int32](repeating: 0, count: n)
        speechCondition = [Float](repeating: 0, count: n * 1024 * 100)
        paddingMask = [Float](repeating: 0, count: n * 1024)
        try luxCheck(fa_luxtts_begin(handle, Int32(n), audio, off, promptTokenCounts, textTokenCounts, speeds, seeds,
                                     &reasons, &ids, &plans, &speechCondition, &paddingMask), "fa_luxtts_begin")
        return (ids, plans)
    }

    /// text_condition [n x 1024 x 100] from the text encoder's stride-padded token_embeds.
    public func textCondition(ids: [Int32], tokenEmbeds: UnsafePointer<Float>, rowStride: Int,
                              requestStride: Int) throws -> [Float] {
        var out = [Float](repeating: 0, count: ids.count * 1024 * 100)
        try luxCheck(fa_luxtts_text_condition(handle, Int32(ids.count), ids, tokenEmbeds, Int64(rowStride),
                                              Int64(requestStride), &out), "fa_luxtts_text_condition")
        return out
    }

    /// The FmDecoder's x [n x 1024 x 100] and t [n].
    public func modelInputs(ids: [Int32]) throws -> (x: [Float], t: [Float]) {
        var x = [Float](repeating: 0, count: ids.count * 1024 * 100)
        var t = [Float](repeating: 0, count: ids.count)
        try luxCheck(fa_luxtts_model_inputs(handle, Int32(ids.count), ids, &x, &t), "fa_luxtts_model_inputs")
        return (x, t)
    }

    /// One anchor-Euler update with the FmDecoder's stride-padded v.
    public func advance(ids: [Int32], v: UnsafePointer<Float>, rowStride: Int, requestStride: Int) throws {
        try luxCheck(fa_luxtts_advance(handle, Int32(ids.count), ids, v, Int64(rowStride), Int64(requestStride)),
                     "fa_luxtts_advance")
    }

    /// The vocoder's mel [n x 100 x bucket] for requests of one bucket.
    public func vocoderInput(ids: [Int32], bucket: Int) throws -> [Float] {
        var out = [Float](repeating: 0, count: ids.count * 100 * bucket)
        try luxCheck(fa_luxtts_vocoder_input(handle, Int32(ids.count), ids, Int32(bucket), &out),
                     "fa_luxtts_vocoder_input")
        return out
    }

    /// Each request's 48 kHz samples; closes the requests.
    public func finish(ids: [Int32], audio: UnsafePointer<Float>, rowStride: Int, rowLength: Int) throws -> [[Float]] {
        var lengths = [Int64](repeating: 0, count: ids.count)
        var total: Int64 = 0
        var out = [Float](repeating: 0, count: ids.count * min(rowLength, 554 * 512))
        try luxCheck(fa_luxtts_finish(handle, Int32(ids.count), ids, audio, Int64(rowStride), Int64(rowLength), &out,
                                      out.count, &lengths, &total), "fa_luxtts_finish")
        var at = 0
        return lengths.map { n in defer { at += Int(n) }; return Array(out[at..<at + Int(n)]) }
    }

    public func close(id: Int32) throws { try luxCheck(fa_luxtts_close(handle, id), "fa_luxtts_close") }
}
