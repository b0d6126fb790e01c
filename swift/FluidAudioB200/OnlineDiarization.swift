// Streaming speaker tracking (Sources/FluidAudio/Diarizer/Core, Clustering) on the GPU (fa_od_*): DiarizerManager's
// chunk logic and SpeakerManager's speaker database for many live sessions, as chunk inputs / embedding inputs /
// advance around the app's segmentation and embedding models, plus the database operations.  The CoreML models stay
// in the app.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func odCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

/// DiarizerConfig as fa_od_config.
public func makeOnlineDiarConfig(clusteringThreshold: Float = 0.7, minSpeechDuration: Float = 1.0,
                                 minActiveFramesCount: Float = 10.0, chunkDuration: Float = 10.0,
                                 chunkOverlap: Float = 0.0) -> fa_od_config {
    fa_od_config(clustering_threshold: clusteringThreshold, min_speech_duration: minSpeechDuration,
                 min_embedding_update_duration: 2.0, min_silence_gap: 0.5, num_clusters: -1,
                 min_active_frames_count: minActiveFramesCount, chunk_duration: chunkDuration,
                 chunk_overlap: chunkOverlap)
}

/// Model inputs for chunks: (segmentation [n x 160000], embedding waveform [n x 160000]).
public func onlineDiarChunkInputs(_ chunks: [[Float]], chunkSize: Int64) throws -> ([Float], [Float]) {
    var off: [Int64] = [0]
    for c in chunks { off.append(off.last! + Int64(c.count)) }
    let audio = chunks.flatMap { $0 }
    var seg = [Float](repeating: 0, count: chunks.count * Int(FA_OD_MODEL_SAMPLES))
    var wave = seg
    try odCheck(fa_od_chunk_inputs(audio, off, Int32(chunks.count), chunkSize, &seg, &wave), "fa_od_chunk_inputs")
    return (seg, wave)
}

/// Live sessions, each one SpeakerManager in HBM (fa_od_databases).  Speakers are (named, key) pairs: named 0 is the
/// canonical decimal id `key`.
public final class SpeakerDatabases {
    let handle: OpaquePointer
    public let frames: Int32
    public var config: fa_od_config

    public init(frames: Int32 = 589, config: fa_od_config = makeOnlineDiarConfig()) throws {
        var h: OpaquePointer?
        try odCheck(fa_od_create(frames, &h), "fa_od_create")
        handle = h!
        self.frames = frames
        self.config = config
    }

    deinit { fa_od_destroy(handle) }

    public func open() throws -> Int32 {
        var id: Int32 = 0
        try odCheck(fa_od_open(handle, &id), "fa_od_open")
        return id
    }

    public func close(_ session: Int32) throws { try odCheck(fa_od_close(handle, session), "fa_od_close") }

    /// logits [n x F x 7] -> (masks [n x 3 x F], need [n x 3])
    public func embeddingInputs(sessions: [Int32], logits: [Float]) throws -> ([Float], [Int32]) {
        var masks = [Float](repeating: 0, count: sessions.count * 3 * Int(frames))
        var need = [Int32](repeating: 0, count: sessions.count * 3)
        var cfg = config
        try odCheck(fa_od_embedding_inputs(handle, Int32(sessions.count), sessions, logits, &cfg, &masks, &need),
                    "fa_od_embedding_inputs")
        return (masks, need)
    }

    /// embeddings [n x 3 x 256] -> (assigned [n x 3 x 2], segment counts, segment ids, segment values)
    public func advance(sessions: [Int32], embeddings: [Float], chunkOffsets: [Double]) throws
        -> ([Int64], [Int32], [Int64], [Float]) {
        let n = sessions.count, bound = 3 * ((Int(frames) + 1) / 2)
        var assigned = [Int64](repeating: 0, count: n * 6)
        var counts = [Int32](repeating: 0, count: n)
        var ids = [Int64](repeating: 0, count: n * bound * 2)
        var values = [Float](repeating: 0, count: n * bound * 3)
        var cfg = config
        try odCheck(fa_od_advance(handle, Int32(n), sessions, embeddings, chunkOffsets, &cfg, &assigned, &counts, &ids,
                                  &values), "fa_od_advance")
        return (assigned, counts, ids, values)
    }

    /// Cosine distances [count x speakers] from embeddings to a session's speakers, in database order.
    public func distances(session: Int32, embeddings: [Float]) throws -> [Float] {
        var count: Int64 = 0, next: Int64 = 0
        try odCheck(fa_od_speaker_count(handle, session, &count, &next), "fa_od_speaker_count")
        let q = embeddings.count / Int(FA_OD_DIM)
        var out = [Float](repeating: 0, count: q * Int(count))
        try odCheck(fa_od_query(handle, session, Int32(q), embeddings, &out), "fa_od_query")
        return out
    }

    public func removeSpeaker(session: Int32, named: Int32, key: Int64, keepIfPermanent: Bool = true) throws -> Bool {
        var done: Int32 = 0
        try odCheck(fa_od_remove(handle, session, named, key, keepIfPermanent ? 1 : 0, &done), "fa_od_remove")
        return done != 0
    }

    public func reset(session: Int32, keepIfPermanent: Bool = false) throws {
        try odCheck(fa_od_reset(handle, session, keepIfPermanent ? 1 : 0), "fa_od_reset")
    }
}
