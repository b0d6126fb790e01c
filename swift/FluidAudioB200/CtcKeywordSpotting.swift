// CTC keyword spotting (CtcKeywordSpotter / CtcDPAlgorithm, ASR/Parakeet/SlidingWindow/CustomVocabulary/WordSpotting/) on
// the GPU (fa_ctc_*): the log-softmax of the CTC logits, the chunk merge of long clips, the CTC-WS dynamic program for every
// vocabulary term in every clip in one call, and the rescorer's constrained queries in one launch.  The CTC model, the
// tokenizers and the term-length filter stay with the caller.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func ctcCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

private func flatten(_ lists: [[Int]]) -> ([Int32], [Int64]) {
    var tokens: [Int32] = []
    var offsets: [Int64] = [0]
    for list in lists {
        tokens.append(contentsOf: list.map { Int32($0) })
        offsets.append(Int64(tokens.count))
    }
    return (tokens, offsets)
}

public enum CtcKeywordSpotting {
    /// applyLogSoftmax / makeLogProbs: `logits` is T × V, time-major, or V × T with `vocabMajor` (the rank-4 CoreML output).
    public static func applyLogSoftmax(logits: [Float], frames: Int, vocabSize: Int, blankId: Int,
                                       temperature: Float = 1.0, blankBias: Float = 0.0,
                                       vocabMajor: Bool = false) throws -> [Float] {
        var out = [Float](repeating: 0, count: frames * vocabSize)
        try ctcCheck(fa_ctc_log_softmax(logits, Int32(frames), Int32(vocabSize),
                                        Int32(vocabMajor ? FA_CTC_LAYOUT_VOCAB_MAJOR.rawValue
                                                         : FA_CTC_LAYOUT_TIME_MAJOR.rawValue),
                                        temperature, blankBias, Int32(blankId), &out), "fa_ctc_log_softmax")
        return out
    }

    /// computeLogProbsChunked's concatenation of per-chunk log-probs (each rows × V, time-major).
    public static func mergeChunks(_ chunks: [[Float]], vocabSize: Int, frameDuration: Double) throws -> [Float] {
        let overlap = Int32(Int(Double(32_000) / Double(16_000) / frameDuration))
        var offsets: [Int64] = [0]
        for c in chunks { offsets.append(offsets.last! + Int64(c.count / vocabSize)) }
        let flat = chunks.flatMap { $0 }
        var out = [Float](repeating: 0, count: flat.count)
        var frames: Int32 = 0
        try ctcCheck(fa_ctc_merge_chunks(flat, offsets, Int32(chunks.count), Int32(vocabSize), overlap, &out,
                                         out.count, &frames), "fa_ctc_merge_chunks")
        return Array(out.prefix(Int(frames) * vocabSize))
    }

    /// ctcWordSpotConstrained for many queries over one clip: (score, startFrame, endFrame) per query.
    public static func wordSpotConstrained(logProbs: [Float], frames: Int, vocabSize: Int, blankId: Int,
                                           queries: [(tokens: [Int], searchStart: Int, searchEnd: Int)]) throws
        -> [(score: Float, startFrame: Int, endFrame: Int)]
    {
        let (tokens, offsets) = flatten(queries.map { $0.tokens })
        let starts = queries.map { Int64($0.searchStart) }, ends = queries.map { Int64($0.searchEnd) }
        var score = [Float](repeating: 0, count: queries.count)
        var a = [Int64](repeating: 0, count: queries.count), b = [Int64](repeating: 0, count: queries.count)
        try ctcCheck(fa_ctc_spot_constrained(logProbs, Int32(frames), Int32(vocabSize), Int32(blankId),
                                             Int32(queries.count), tokens, offsets, starts, ends, &score, &a, &b),
                     "fa_ctc_spot_constrained")
        return (0..<queries.count).map { (score[$0], Int(a[$0]), Int(b[$0])) }
    }
}

/// A vocabulary of token-id terms in HBM: ctcWordSpotMultiple for every term in many clips per call.
public final class CtcVocabularySpotter {
    public struct Detection {
        public var clip: Int, term: Int
        public var score: Float
        public var startFrame: Int, endFrame: Int
    }

    private var handle: OpaquePointer?
    public let vocabSize: Int
    public let termCount: Int

    /// `terms` are `ctcTokenIds ?? tokenIds` of the terms that pass the length filter (at most 127 tokens each).
    public init(vocabSize: Int, blankId: Int, terms: [[Int]]) throws {
        let (tokens, offsets) = flatten(terms)
        var h: OpaquePointer?
        try ctcCheck(fa_ctc_spotter_create(Int32(vocabSize), Int32(blankId), Int32(terms.count), tokens, offsets, &h),
                     "fa_ctc_spotter_create")
        handle = h
        self.vocabSize = vocabSize
        termCount = terms.count
    }

    deinit { fa_ctc_spotter_destroy(handle) }

    /// spotKeywordsFromLogProbs without the text filter: clip b's log-probs are clips[b] (T_b × V, time-major).
    public func spot(clips: [[Float]], minScore: Float? = nil) throws -> [Detection] {
        var offsets: [Int64] = [0]
        for c in clips { offsets.append(offsets.last! + Int64(c.count / vocabSize)) }
        let flat = clips.flatMap { $0 }
        var counts = [Int64](repeating: 0, count: clips.count * termCount)
        var total: Int64 = 0
        var out = [fa_ctc_detection](repeating: fa_ctc_detection(), count: max(1, flat.count / vocabSize / 8))
        var base = minScore ?? 0
        func call() -> fa_status {
            withUnsafePointer(to: &base) { ms in
                fa_ctc_spot(handle, flat, offsets, Int32(clips.count), minScore == nil ? nil : ms, &counts, &total,
                            &out, out.count)
            }
        }
        var status = call()
        if status == FA_STATUS_OUTPUT_TOO_SMALL {
            out = [fa_ctc_detection](repeating: fa_ctc_detection(), count: Int(total))
            status = call()
        }
        try ctcCheck(status, "fa_ctc_spot")
        return out.prefix(Int(total)).map {
            Detection(clip: Int($0.clip), term: Int($0.term), score: $0.score, startFrame: Int($0.start_frame),
                      endFrame: Int($0.end_frame))
        }
    }
}
