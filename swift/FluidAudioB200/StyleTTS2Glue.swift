// StyleTTS2 synthesis glue (Sources/FluidAudio/TTS/StyleTTS2/Pipeline/Synthesize/StyleTTS2Synthesizer.swift) on the
// GPU (fa_styletts2_*): the host work between the eight models for many requests per call.  The CoreML models stay in
// the app.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func styleCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

public enum StyleTTS2Glue {
    /// fa_styletts2_plan: the bert / sampler bucket (57, 64, 128, 256) and the reason code (0 when it has one).
    public static func plan(tokenCount: Int) throws -> (bucket: Int, reason: Int) {
        var bucket: Int32 = 0
        var reason: Int32 = 0
        try styleCheck(fa_styletts2_plan(Int32(tokenCount), &bucket, &reason), "fa_styletts2_plan")
        return (Int(bucket), Int(reason))
    }

    /// bert's padded tokens and attention mask [n x bucket] and the fused sampler's noise [n x 5 x 256] (row 0
    /// noise_init, rows 1 ... 4 noises_aux) for requests of one bucket.
    public static func samplerInputs(tokenIds: [[Int32]], seeds: [UInt64], bucket: Int) throws
        -> (tokens: [Int32], attentionMask: [Int32], noise: [Float])
    {
        let n = tokenIds.count
        var offsets: [Int64] = [0]
        for t in tokenIds { offsets.append(offsets.last! + Int64(t.count)) }
        let flat = tokenIds.flatMap { $0 }
        var tokens = [Int32](repeating: 0, count: n * bucket)
        var mask = [Int32](repeating: 0, count: n * bucket)
        var noise = [Float](repeating: 0, count: n * 5 * 256)
        var reasons = [Int32](repeating: 0, count: n)
        try styleCheck(fa_styletts2_sampler_inputs(Int32(n), flat, offsets, seeds, Int32(bucket), &tokens, &mask,
                                                   &noise, &reasons), "fa_styletts2_sampler_inputs")
        return (tokens, mask, noise)
    }

    /// blendStyle for n requests: sPred and refS [n x 256] -> (ref, s) [n x 128].
    public static func blendStyle(sPred: [Float], refS: [Float], alphas: [Float], betas: [Float]) throws
        -> (ref: [Float], s: [Float])
    {
        let n = alphas.count
        var ref = [Float](repeating: 0, count: n * 128)
        var s = [Float](repeating: 0, count: n * 128)
        try styleCheck(fa_styletts2_style(Int32(n), sPred, refS, alphas, betas, &ref, &s), "fa_styletts2_style")
        return (ref, s)
    }

    /// Durations and the duration-aligned en [n x dC x frameStride] and asr [n x tC x frameStride] from each
    /// request's logits [tokens x C], d [tokens x dC] and tEn [tC x tokens], packed with the strides given.
    /// Throws FA_STATUS_OUTPUT_TOO_SMALL with `frames` filled when a request has more frames than frameStride.
    public static func align(tokenCounts: [Int32], logits: [Float], logitChannels: Int, logitRowStride: Int,
                             logitRequestStride: Int, d: [Float], dChannels: Int, dRowStride: Int,
                             dRequestStride: Int, tEn: [Float], tEnChannels: Int, tEnRowStride: Int,
                             tEnRequestStride: Int, frameStride: Int, frames: inout [Int64])
        throws -> (en: [Float], asr: [Float], durations: [Int32])
    {
        let n = tokenCounts.count
        var en = [Float](repeating: 0, count: n * dChannels * frameStride)
        var asr = [Float](repeating: 0, count: n * tEnChannels * frameStride)
        var durations = [Int32](repeating: 0, count: Int(tokenCounts.reduce(0, +)))
        var reasons = [Int32](repeating: 0, count: n)
        frames = [Int64](repeating: 0, count: n)
        try styleCheck(fa_styletts2_align(Int32(n), tokenCounts, logits, Int32(logitChannels), Int64(logitRowStride),
                                          Int64(logitRequestStride), d, Int32(dChannels), Int64(dRowStride),
                                          Int64(dRequestStride), tEn, Int32(tEnChannels), Int64(tEnRowStride),
                                          Int64(tEnRequestStride), Int64(frameStride), &en, &asr, &frames,
                                          &durations, &reasons), "fa_styletts2_align")
        return (en, asr, durations)
    }
}
