// Sortformer's streaming state (Sources/FluidAudio/Diarizer/Sortformer/SortformerStateUpdater.swift, the state of
// SortformerTypes.swift:270-327 and the padded inputs of SortformerModelInference.swift:266-303) for many live sessions
// in HBM (fa_sortformer_*).  SortformerStateUpdater.streamingUpdate becomes `update([id: output])`, and the copies of
// runMainModel become `modelInputs([id])`; a server ticking thousands of sessions passes them all in one call: one
// kernel launch per update, one per model-input gather, one synchronisation each.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public final class SortformerStreams {
    public struct ModelOutput {
        /// chunk_pre_encoder_embs [embLength * 512] and speaker_preds [predRows * 4] (probabilities)
        public var chunkEmbeddings: [Float]
        public var predictions: [Float]
        /// nil: the streaming rule (chunk index > 0 ? chunkLeftContext : 0) and chunkRightContext
        public var leftContext: Int32? = nil
        public var rightContext: Int32? = nil
    }

    private var handle: OpaquePointer?
    private var chunks: [Int32: Int] = [:]   // chunk index of each open session, for the streaming rule
    public let config: fa_sortformer_config

    /// `preset`: FA_SORTFORMER_DEFAULT ... FA_SORTFORMER_EFFICIENT_V2_1; maxCoreFrames 0 = chunkLen.
    public init(preset: Int32 = Int32(FA_SORTFORMER_DEFAULT), maxCoreFrames: Int32 = 0) {
        var c = fa_sortformer_config()
        precondition(fa_sortformer_default_config(&c, preset) == FA_STATUS_OK)
        var h: OpaquePointer?
        let status = fa_sortformer_create(&c, maxCoreFrames, &h)
        precondition(status == FA_STATUS_OK, "fa_sortformer_create: \(String(cString: fa_last_error()))")
        handle = h
        config = c
    }

    deinit { fa_sortformer_destroy(handle) }

    /// SortformerStreamingState(config:): a new session (the lowest free id).
    public func open() -> Int32 {
        var id: Int32 = -1
        let status = fa_sortformer_open(handle, &id)
        precondition(status == FA_STATUS_OK, "fa_sortformer_open: \(String(cString: fa_last_error()))")
        chunks[id] = 0
        return id
    }

    public func close(_ session: Int32) {
        _ = fa_sortformer_close(handle, session)
        chunks[session] = nil
    }

    /// The streaming rule of SortformerDiarizer.swift:553: no left context on a session's first chunk.
    private func streamingLeftContext(_ session: Int32) -> Int32 {
        (chunks[session] ?? 0) > 0 ? config.chunk_left_context : 0
    }

    /// streamingUpdate for every session in `outputs`; returns each session's (confirmed, tentative) rows [frames * 4].
    public func update(_ outputs: [Int32: ModelOutput]) throws -> [Int32: (confirmed: [Float], tentative: [Float])] {
        let ids = Array(outputs.keys)
        let embRows = ids.map { outputs[$0]!.chunkEmbeddings.count / 512 }.max() ?? 0
        let predRows = ids.map { outputs[$0]!.predictions.count / 4 }.max() ?? 0
        var embs = [Float](repeating: 0, count: ids.count * embRows * 512)
        var preds = [Float](repeating: 0, count: ids.count * predRows * 4)
        for (i, id) in ids.enumerated() {
            let o = outputs[id]!
            embs.replaceSubrange((i * embRows * 512)..<(i * embRows * 512 + o.chunkEmbeddings.count), with: o.chunkEmbeddings)
            preds.replaceSubrange((i * predRows * 4)..<(i * predRows * 4 + o.predictions.count), with: o.predictions)
        }
        let lengths = ids.map { Int32(outputs[$0]!.chunkEmbeddings.count / 512) }
        let explicit = ids.contains { outputs[$0]!.leftContext != nil || outputs[$0]!.rightContext != nil }
        let lc: [Int32]? = explicit ? ids.map { outputs[$0]!.leftContext ?? streamingLeftContext($0) } : nil
        let rc: [Int32]? = explicit ? ids.map { outputs[$0]!.rightContext ?? config.chunk_right_context } : nil
        let cap = max(1, ids.count * embRows * 4)
        var confirmed = [Float](repeating: 0, count: cap), tentative = [Float](repeating: 0, count: cap)
        var cRows = [Int64](repeating: 0, count: ids.count), tRows = [Int64](repeating: 0, count: ids.count)
        let status = fa_sortformer_update(handle, Int32(ids.count), ids, embs, Int32(embRows), preds, Int32(predRows),
                                          lengths, lc, rc, &confirmed, cap, &tentative, cap, &cRows, &tRows)
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fa_sortformer_update", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        for id in ids { chunks[id, default: 0] += 1 }
        var result: [Int32: (confirmed: [Float], tentative: [Float])] = [:]
        var c = 0, t = 0
        for (i, id) in ids.enumerated() {
            let nc = Int(cRows[i]) * 4, nt = Int(tRows[i]) * 4
            result[id] = (Array(confirmed[c..<(c + nc)]), Array(tentative[t..<(t + nt)]))
            c += nc
            t += nt
        }
        return result
    }

    /// runMainModel's spkcache [spkcacheLen * 512] and fifo [fifoLen * 512] inputs, zero padded, with their lengths.
    public func modelInputs(_ sessions: [Int32]) -> [(spkcache: [Float], spkcacheLength: Int32, fifo: [Float], fifoLength: Int32)] {
        let cacheFloats = Int(config.spkcache_len) * 512, fifoFloats = Int(config.fifo_len) * 512
        var sc = [Float](repeating: 0, count: max(1, sessions.count * cacheFloats))
        var ff = [Float](repeating: 0, count: max(1, sessions.count * fifoFloats))
        var sl = [Int32](repeating: 0, count: sessions.count), fl = [Int32](repeating: 0, count: sessions.count)
        let status = fa_sortformer_model_inputs(handle, Int32(sessions.count), sessions, &sc, &ff, &sl, &fl)
        precondition(status == FA_STATUS_OK, "fa_sortformer_model_inputs: \(String(cString: fa_last_error()))")
        return sessions.indices.map { i in
            (Array(sc[(i * cacheFloats)..<((i + 1) * cacheFloats)]), sl[i],
             Array(ff[(i * fifoFloats)..<((i + 1) * fifoFloats)]), fl[i])
        }
    }
}
