// DiarizerTimeline's numeric core (Sources/FluidAudio/Diarizer/DiarizerTimeline.swift) for many live sessions in HBM
// (fa_diarizer_timeline_*).  DiarizerTimeline.addChunk becomes `push([id: (finalized, tentative)])`, which returns each
// session's new segments; the speakers, their names and their segment lists stay in the caller's DiarizerTimeline, which
// appends these segments as commitSegment does.  A server ticking thousands of sessions passes them all in one call: two
// kernel launches and at most two synchronisations per push.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public final class DiarizerTimelines {
    public struct Segment {
        public var speakerIndex: Int
        public var startFrame: Int
        public var endFrame: Int
        public var activity: Float
    }

    private var handle: OpaquePointer?
    public let config: fa_diarizer_timeline_config
    public let maxTentativeRows: Int32

    /// `preset`: FA_TIMELINE_PRESET_SORTFORMER (sortformerDefault) or FA_TIMELINE_PRESET_DEFAULT with numSpeakers and
    /// frameDurationSeconds (LS-EEND: maxSpeakers, 0.1 s); maxStoredFrames caps the finalized rows kept per session.
    public init(preset: Int32 = Int32(FA_TIMELINE_PRESET_SORTFORMER), numSpeakers: Int32 = 4,
                frameDurationSeconds: Float = 0.08, maxStoredFrames: Int32 = Int32(FA_TIMELINE_DEFAULT_STORED_FRAMES),
                maxTentativeRows: Int32 = 64) {
        var c = fa_diarizer_timeline_config()
        precondition(fa_diarizer_timeline_default_config(&c, preset, numSpeakers, frameDurationSeconds) == FA_STATUS_OK)
        c.max_stored_frames = maxStoredFrames
        var h: OpaquePointer?
        let status = fa_diarizer_timeline_create(&c, maxTentativeRows, &h)
        precondition(status == FA_STATUS_OK, "fa_diarizer_timeline_create: \(String(cString: fa_last_error()))")
        handle = h
        config = c
        self.maxTentativeRows = maxTentativeRows
    }

    deinit { fa_diarizer_timeline_destroy(handle) }

    /// DiarizerTimeline(config:): a new session (the lowest free id).
    public func open() -> Int32 {
        var id: Int32 = -1
        let status = fa_diarizer_timeline_open(handle, &id)
        precondition(status == FA_STATUS_OK, "fa_diarizer_timeline_open: \(String(cString: fa_last_error()))")
        return id
    }

    public func close(_ session: Int32) { _ = fa_diarizer_timeline_close(handle, session) }

    /// addChunk for every session in `chunks` (rows [frames * numSpeakers]); returns each session's new finalized and
    /// tentative segments, speaker-major and in frame order within a speaker.
    public func push(_ chunks: [Int32: (finalized: [Float], tentative: [Float])]) throws
        -> [Int32: (finalized: [Segment], tentative: [Segment])]
    {
        let ids = Array(chunks.keys)
        let S = Int(config.num_speakers)
        let fRows = ids.map { Int64(chunks[$0]!.finalized.count / S) }
        let tRows = ids.map { Int64(chunks[$0]!.tentative.count / S) }
        let fin = ids.flatMap { chunks[$0]!.finalized }, ten = ids.flatMap { chunks[$0]!.tentative }
        var fBound: Int64 = 0, tBound: Int64 = 0
        _ = fa_diarizer_timeline_segment_bound(config.num_speakers, Int32(ids.count), fRows, tRows, &fBound, &tBound)
        var fOut = [fa_diarizer_timeline_segment](repeating: .init(), count: max(1, Int(fBound)))
        var tOut = [fa_diarizer_timeline_segment](repeating: .init(), count: max(1, Int(tBound)))
        var fCounts = [Int64](repeating: 0, count: ids.count), tCounts = [Int64](repeating: 0, count: ids.count)
        let status = fa_diarizer_timeline_push(handle, Int32(ids.count), ids, fin, fRows, ten, tRows, &fOut, Int(fBound),
                                               &tOut, Int(tBound), &fCounts, &tCounts)
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fa_diarizer_timeline_push", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        let convert = { (s: fa_diarizer_timeline_segment) in
            Segment(speakerIndex: Int(s.speaker), startFrame: Int(s.start_frame), endFrame: Int(s.end_frame),
                    activity: s.activity)
        }
        var result: [Int32: (finalized: [Segment], tentative: [Segment])] = [:]
        var f = 0, t = 0
        for (i, id) in ids.enumerated() {
            let nf = Int(fCounts[i]), nt = Int(tCounts[i])
            result[id] = (fOut[f..<(f + nf)].map(convert), tOut[t..<(t + nt)].map(convert))
            f += nf
            t += nt
        }
        return result
    }

    /// finalize (:877-891) for these sessions: their tentative rows become finalized.  The caller's speakers move their
    /// tentative segments to the finalized ones.
    public func finalize(_ sessions: [Int32]) {
        precondition(fa_diarizer_timeline_finalize(handle, Int32(sessions.count), sessions) == FA_STATUS_OK)
    }

    /// reset (:897-934): no predictions, cursor 0, fresh scratches.
    public func reset(_ sessions: [Int32]) {
        precondition(fa_diarizer_timeline_reset(handle, Int32(sessions.count), sessions) == FA_STATUS_OK)
    }

    /// removeSpeaker(clearCurrentSegment: true) / upsertSpeaker(transferCurrentSegment: false): a fresh scratch.
    public func clearSpeaker(_ session: Int32, slot: Int32) {
        precondition(fa_diarizer_timeline_clear_speaker(handle, session, slot) == FA_STATUS_OK)
    }

    /// finalizedPredictions (the last maxStoredFrames finalized rows), tentativePredictions and numFinalizedFrames.
    public func predictions(_ session: Int32) -> (finalized: [Float], tentative: [Float], numFinalizedFrames: Int) {
        let S = Int(config.num_speakers)
        var info = fa_diarizer_timeline_session_info()
        var stored = [Float](repeating: 0, count: max(1, Int(config.max_stored_frames) * S))
        var tent = [Float](repeating: 0, count: max(1, Int(maxTentativeRows) * S))
        precondition(fa_diarizer_timeline_session_state(handle, session, &info, &stored, &tent, nil) == FA_STATUS_OK)
        return (Array(stored[0..<(Int(info.stored_frames) * S)]), Array(tent[0..<(Int(info.tentative_frames) * S)]),
                Int(info.finalized_frames))
    }
}
