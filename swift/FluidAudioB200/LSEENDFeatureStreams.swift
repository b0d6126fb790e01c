// LSEENDFeatureProvider (Sources/FluidAudio/Diarizer/LS-EEND/LSEENDPreprocessor.swift:46-384) for many live sessions in
// HBM (fa_lseend_stream_*).  enqueueAudio, drainRightContextWithSilence and the emitNextChunk loop of LSEENDDiarizer
// become `push([id: samples], drain:)`, which returns every chunk each session made ready: its mel features
// [melFrames x nMels], decoder-mask window and warm-up count, in order, for the caller's LS-EEND model.  The model and its
// recurrent state stay with the caller.  A server ticking thousands of sessions passes them all in one call: four kernel
// launches and one synchronisation per push.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public final class LSEENDFeatureStreams {
    public struct Chunk {
        public var melFeatures: [Float]     // melFrames * nMels, time-major
        public var decoderMask: [Float]     // chunkSize
        public var warmupFrames: Int
    }

    private var handle: OpaquePointer?
    public let config: fa_lseend_stream_config
    public let sizes: fa_lseend_stream_sizes

    /// The LSEENDMetadata fields the provider reads; audio must arrive at `sampleRate` (resample with fa_audio_resample).
    public init(sampleRate: Int32, nMels: Int32, hopLength: Int32, winLength: Int32, contextSize: Int32,
                subsampling: Int32, chunkSize: Int32, convDelay: Int32,
                precision: Int32 = Int32(FA_MEL_PRECISION_F64)) throws {
        var c = fa_lseend_stream_config(sample_rate: sampleRate, n_mels: nMels, hop_length: hopLength,
                                         win_length: winLength, context_size: contextSize, subsampling: subsampling,
                                         chunk_size: chunkSize, conv_delay: convDelay, precision: precision)
        var s = fa_lseend_stream_sizes()
        var h: OpaquePointer?
        var status = fa_lseend_stream_resolve(&c, &s)
        if status == FA_STATUS_OK { status = fa_lseend_stream_create(&c, &h) }
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fa_lseend_stream_create", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        handle = h
        config = c
        sizes = s
    }

    deinit { fa_lseend_stream_destroy(handle) }

    /// LSEENDFeatureProvider(from:): a new session (the lowest free id).
    public func open() -> Int32 {
        var id: Int32 = -1
        let status = fa_lseend_stream_open(handle, &id)
        precondition(status == FA_STATUS_OK, "fa_lseend_stream_open: \(String(cString: fa_last_error()))")
        return id
    }

    public func close(_ session: Int32) { _ = fa_lseend_stream_close(handle, session) }

    /// enqueueAudio for every session in `audio`, drainRightContextWithSilence for those in `drain`, then emitNextChunk
    /// until none is ready.  Returns each named session's chunks in order.
    public func push(_ audio: [Int32: [Float]], drain: Set<Int32> = []) throws -> [Int32: [Chunk]] {
        let ids = Array(Set(audio.keys).union(drain))
        var offsets = [Int64](repeating: 0, count: ids.count + 1)
        for (i, id) in ids.enumerated() { offsets[i + 1] = offsets[i] + Int64(audio[id]?.count ?? 0) }
        let samples = ids.flatMap { audio[$0] ?? [] }
        let drains = ids.map { drain.contains($0) ? Int32(1) : Int32(0) }
        let total = ids.enumerated().reduce(0) { acc, e in
            acc + Int(fa_lseend_stream_chunks(handle, e.element, offsets[e.offset + 1] - offsets[e.offset], drains[e.offset]))
        }
        let F = Int(sizes.mel_frames) * Int(config.n_mels), T = Int(config.chunk_size)
        var features = [Float](repeating: 0, count: max(1, total * F))
        var masks = [Float](repeating: 0, count: max(1, total * T))
        var warmup = [Int32](repeating: 0, count: max(1, total))
        var counts = [Int64](repeating: 0, count: ids.count)
        let status = fa_lseend_stream_push(handle, Int32(ids.count), ids, samples, offsets, drains, &features,
                                           features.count, &masks, masks.count, &warmup, warmup.count, &counts)
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fa_lseend_stream_push", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        var result: [Int32: [Chunk]] = [:]
        var c = 0
        for (i, id) in ids.enumerated() {
            result[id] = (c..<(c + Int(counts[i]))).map { k in
                Chunk(melFeatures: Array(features[(k * F)..<((k + 1) * F)]), decoderMask: Array(masks[(k * T)..<((k + 1) * T)]),
                      warmupFrames: Int(warmup[k]))
            }
            c += Int(counts[i])
        }
        return result
    }

    /// takeSnapshot (:206-218) for these sessions; one snapshot per session, replacing an earlier one.
    public func takeSnapshot(_ sessions: [Int32]) {
        precondition(fa_lseend_stream_snapshot(handle, Int32(sessions.count), sessions) == FA_STATUS_OK)
    }

    /// rollback(to:) (:224-233) to each session's snapshot; the snapshot stays.
    public func rollback(_ sessions: [Int32]) throws {
        let status = fa_lseend_stream_rollback(handle, Int32(sessions.count), sessions)
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fa_lseend_stream_rollback", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
    }

    /// reset (:236-245): fresh queues, a zero running mean, decoderMaskEnd 0.
    public func reset(_ sessions: [Int32]) {
        precondition(fa_lseend_stream_reset(handle, Int32(sessions.count), sessions) == FA_STATUS_OK)
    }
}
