// The incremental mel stream of Sources/FluidAudio/Diarizer/Sortformer/SortformerDiarizer.swift (resetMelStreamLocked
// :204-217, addAudio :417-424, preprocessAudioToFeaturesLocked / emitMelFramesLocked :842-870,
// padAndEmitRemainingMelLocked :876-901) for many live sessions on one AudioMelSpectrogram handle (fa_mel_stream_*).
// SortformerDiarizer.preprocessAudioToFeaturesLocked becomes `push([id: samples])` and padAndEmitRemainingMelLocked
// becomes `push([id: []], finish: [id])`; the returned rows are what emitMelFramesLocked appends to featureBuffer.
// A server ticking thousands of sessions pushes them all in one call: two kernel launches and one synchronisation.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public final class MelStreams {
    private let mel: AudioMelSpectrogram
    private let nMels: Int

    /// The handle's configuration must have padTo <= 1 and hopLength <= winLength.
    public init(_ mel: AudioMelSpectrogram) {
        self.mel = mel
        self.nMels = mel.melBins
    }

    /// resetMelStreamLocked: a new session (the lowest free id) with nFFT/2 zeros buffered.
    public func open() -> Int32 {
        var id: Int32 = -1
        let status = fa_mel_stream_open(mel.rawHandle, &id)
        precondition(status == FA_STATUS_OK, "fa_mel_stream_open: \(String(cString: fa_last_error()))")
        return id
    }

    public func close(_ session: Int32) { _ = fa_mel_stream_close(mel.rawHandle, session) }

    /// Mel frames the next push of `samples` (and `finish`) to `session` emits.
    public func pendingFrames(_ session: Int32, samples: Int, finish: Bool = false) -> Int {
        Int(fa_mel_stream_frames(mel.rawHandle, session, Int64(samples), finish ? 1 : 0))
    }

    /// addAudio for every session in `chunks`, then finalizeSession for those in `finish` (after their samples).
    /// Returns each session's new frames, time-major [frames * nMels].
    public func push(_ chunks: [Int32: [Float]], finish: Set<Int32> = []) -> [Int32: [Float]] {
        let ids = Array(chunks.keys) + finish.subtracting(chunks.keys).sorted()
        var offsets: [Int64] = [0]
        var audio: [Float] = []
        for id in ids {
            audio.append(contentsOf: chunks[id] ?? [])
            offsets.append(Int64(audio.count))
        }
        let fin: [Int32] = ids.map { finish.contains($0) ? 1 : 0 }
        let rows = ids.indices.reduce(0) { acc, i in
            acc + pendingFrames(ids[i], samples: Int(offsets[i + 1] - offsets[i]), finish: fin[i] != 0)
        }
        var out = [Float](repeating: 0, count: max(1, rows) * nMels)
        var frames = [Int64](repeating: 0, count: ids.count)
        let status = out.withUnsafeMutableBufferPointer { dst in
            fa_mel_stream_push(mel.rawHandle, Int32(ids.count), ids, audio, offsets, fin, dst.baseAddress, dst.count,
                               &frames)
        }
        precondition(status == FA_STATUS_OK, "fa_mel_stream_push: \(String(cString: fa_last_error()))")
        var result: [Int32: [Float]] = [:]
        var row = 0
        for (i, id) in ids.enumerated() {
            let n = Int(frames[i])
            result[id] = Array(out[(row * nMels)..<((row + n) * nMels)])
            row += n
        }
        return result
    }
}
