// Offline Sortformer windows (Sources/FluidAudio/Diarizer/Sortformer/Offline/OfflineSortformerDiarizer.swift) on the
// GPU (fa_offline_sortformer_*): every window of many files as one model batch, then the cross-window speaker
// stitching of all files in one launch.  The CoreML model stays in the app.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func offlineCheck(_ status: fa_status, _ entry: String) throws {
    guard status == FA_STATUS_OK else {
        throw NSError(domain: entry, code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}

public enum OfflineSortformerWindows {
    /// Each file's window count and output rows (ceil(melFrames / 8)) at `overlap` output frames, clamped to 0 ... 383.
    public static func plan(melFrames: [Int64], overlap: Int = 100) throws -> (windows: [Int64], outputFrames: [Int64]) {
        var windows = [Int64](repeating: 0, count: melFrames.count)
        var rows = [Int64](repeating: 0, count: melFrames.count)
        try offlineCheck(fa_offline_sortformer_plan(Int32(overlap), Int32(melFrames.count), melFrames, &windows, &rows),
                         "fa_offline_sortformer_plan")
        return (windows, rows)
    }

    /// runOffline's model inputs for every window of the files whose time-major mel rows start at `melOffsets`
    /// (floats) in `mel`: mel [W x 128 x 3072] channels-first and mel_length [W].
    public static func modelInputs(mel: [Float], melOffsets: [Int64], melFrames: [Int64], overlap: Int = 100) throws
        -> (mel: [Float], melLength: [Int32])
    {
        let w = Int(try plan(melFrames: melFrames, overlap: overlap).windows.reduce(0, +))
        var out = [Float](repeating: 0, count: w * 128 * 3072)
        var lengths = [Int32](repeating: 0, count: w)
        try offlineCheck(fa_offline_sortformer_model_inputs(Int32(overlap), Int32(melFrames.count), mel, melOffsets,
                                                            melFrames, Int64(w), &out, &lengths),
                         "fa_offline_sortformer_model_inputs")
        return (out, lengths)
    }

    /// processComplete's stitching of the model's speaker_preds [W x 384 x 4]: the finalized predictions of every
    /// file [sum of outputFrames x 4], packed in file order, and each window's mapping[windowColumn] = globalSpeaker.
    public static func stitch(speakerPreds: [Float], melFrames: [Int64], overlap: Int = 100) throws
        -> (predictions: [Float], mappings: [Int32])
    {
        let p = try plan(melFrames: melFrames, overlap: overlap)
        var predictions = [Float](repeating: 0, count: Int(p.outputFrames.reduce(0, +)) * 4)
        var mappings = [Int32](repeating: 0, count: Int(p.windows.reduce(0, +)) * 4)
        try offlineCheck(fa_offline_sortformer_stitch(Int32(overlap), Int32(melFrames.count), melFrames, speakerPreds,
                                                      &predictions, &mappings), "fa_offline_sortformer_stitch")
        return (predictions, mappings)
    }
}
