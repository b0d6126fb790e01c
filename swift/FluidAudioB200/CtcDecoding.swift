// CTC decoding (ctcGreedyDecode / ctcBeamSearch with ARPALanguageModel, ASR/Parakeet/SlidingWindow/CTC/) on the GPU
// (fa_ctc_greedy, fa_ctc_beam_search): many clips per call, ids back per clip.  decodeCtcTokenIds and ARPA loading stay
// in the app; an ARPALanguageModel's dictionaries are handed to CtcLanguageModel once.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func decodeCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

private func blob(_ strings: [String]) -> ([CChar], [Int64]) {
    var bytes: [CChar] = []
    var offsets: [Int64] = [0]
    for s in strings {
        bytes.append(contentsOf: s.utf8.map { CChar(bitPattern: $0) })
        offsets.append(Int64(bytes.count))
    }
    bytes.append(0)
    return (bytes, offsets)
}

private func split(_ tokens: [Int32], _ lengths: [Int64]) -> [[Int]] {
    var out: [[Int]] = []
    var at = 0
    for n in lengths {
        out.append(tokens[at..<at + Int(n)].map { Int($0) })
        at += Int(n)
    }
    return out
}

/// An ARPA bigram LM in HBM (fa_ctc_lm): unigrams and bigrams in natural log, as ARPALanguageModel holds them.
public final class CtcLanguageModel {
    let handle: OpaquePointer

    public init(unigrams: [String: (logProb: Float, backoff: Float)], bigrams: [String: [String: Float]]) throws {
        var words = Array(unigrams.keys)
        var index = [String: Int32]()
        for (i, w) in words.enumerated() { index[w] = Int32(i) }
        for (ctx, row) in bigrams {
            for w in [ctx] + Array(row.keys) where index[w] == nil {
                index[w] = Int32(words.count)
                words.append(w)
            }
        }
        let (bytes, offsets) = blob(words)
        let has = words.map { unigrams[$0] != nil ? Int32(1) : 0 }
        let lp = words.map { unigrams[$0]?.logProb ?? 0 }, bo = words.map { unigrams[$0]?.backoff ?? 0 }
        var ctx: [Int32] = [], word: [Int32] = [], blp: [Float] = []
        for (c, row) in bigrams {
            for (w, p) in row {
                ctx.append(index[c]!)
                word.append(index[w]!)
                blp.append(p)
            }
        }
        var h: OpaquePointer?
        try decodeCheck(fa_ctc_lm_create(Int32(words.count), bytes, offsets, has, lp, bo, Int64(ctx.count), ctx, word,
                                         blp, &h), "fa_ctc_lm_create")
        handle = h!
    }

    deinit { fa_ctc_lm_destroy(handle) }
}

/// A vocabulary's pieces in HBM (fa_ctc_decoder) and its decoding calls.
public final class CtcDecoding {
    let handle: OpaquePointer
    public let vocabSize: Int, blankId: Int

    public init(vocabulary: [Int: String], vocabSize: Int, blankId: Int = 1024) throws {
        self.vocabSize = vocabSize
        self.blankId = blankId
        let (bytes, offsets) = blob((0..<vocabSize).map { vocabulary[$0] ?? "" })
        var h: OpaquePointer?
        try decodeCheck(fa_ctc_decoder_create(Int32(vocabSize), Int32(blankId), bytes, offsets, &h),
                        "fa_ctc_decoder_create")
        handle = h!
    }

    deinit { fa_ctc_decoder_destroy(handle) }

    private func flat(_ clips: [[Float]]) -> ([Float], [Int64]) {
        var offsets: [Int64] = [0]
        for c in clips { offsets.append(offsets.last! + Int64(c.count / vocabSize)) }
        return (clips.flatMap { $0 }, offsets)
    }

    /// ctcGreedyDecode's ids for every clip (each T × vocabSize, time-major).
    public func greedy(_ clips: [[Float]]) throws -> [[Int]] {
        let (lp, offsets) = flat(clips)
        var lengths = [Int64](repeating: 0, count: clips.count)
        var tokens = [Int32](repeating: 0, count: max(1, Int(offsets.last!)))
        var total: Int64 = 0
        try decodeCheck(fa_ctc_greedy(lp, offsets, Int32(clips.count), Int32(vocabSize), Int32(blankId), &lengths,
                                      &tokens, tokens.count, &total), "fa_ctc_greedy")
        return split(tokens, lengths)
    }

    /// ctcBeamSearch's best prefix and its total for every clip; the reference's defaults.
    public func beamSearch(_ clips: [[Float]], lm: CtcLanguageModel? = nil, beamWidth: Int = 100,
                           lmWeight: Float = 0.3, wordBonus: Float = 0.0, tokenCandidates: Int = 40) throws
        -> [(ids: [Int], score: Float)]
    {
        let (lp, offsets) = flat(clips)
        var cfg = fa_ctc_beam_config(beam_width: Int32(beamWidth), token_candidates: Int32(tokenCandidates),
                                     lm_weight: lmWeight, word_bonus: wordBonus)
        var lengths = [Int64](repeating: 0, count: clips.count)
        var scores = [Float](repeating: 0, count: clips.count)
        var tokens = [Int32](repeating: 0, count: max(1, Int(offsets.last!)))
        var total: Int64 = 0
        try decodeCheck(fa_ctc_beam_search(handle, lm?.handle, lp, offsets, Int32(clips.count), &cfg, &lengths,
                                           &scores, &tokens, tokens.count, &total), "fa_ctc_beam_search")
        return Array(zip(split(tokens, lengths), scores)).map { (ids: $0.0, score: $0.1) }
    }
}
