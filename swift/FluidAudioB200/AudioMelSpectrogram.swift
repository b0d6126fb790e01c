// Drop-in for Sources/FluidAudio/Shared/AudioMelSpectrogram.swift (same public surface: init :59-70,
// compute :132, computeFlat :185, computeFlatTransposed :299/:325, getFilterbank/getHannWindow :486-493, nFFT).
// All arithmetic happens in libfluidaudio_b200.so on an sm_90a GPU; this file only marshals buffers.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public final class AudioMelSpectrogram {
    public enum PaddingMode: Sendable { case center, prePadded }
    public enum LogFloorMode: Sendable { case additive, clamped }

    public let nFFT: Int
    internal let preemph: Float
    private let nMels: Int
    private let padTo: Int
    private let winLength: Int
    private var handle: OpaquePointer?
    internal var rawHandle: OpaquePointer? { handle }   // for the fused AudioConverter + mel entry (AudioConverter.swift)
    internal var melBins: Int { nMels }
    /// Transform arithmetic: false (default) = FP64 transform rounded once; true = float32 transform like vDSP_DFT
    /// (fa_mel_set_precision, ~1.4x the throughput).  Not part of the reference class.
    public var float32Transform: Bool = false {
        didSet { _ = fa_mel_set_precision(handle, float32Transform ? 1 : 0) }
    }

    public init(
        sampleRate: Int = 16000, nMels: Int = 128, nFFT: Int = 512, hopLength: Int = 160, winLength: Int = 400,
        preemph: Float = 0.97, padTo: Int = 0, logFloor: Float = powf(2, -24),
        logFloorMode: LogFloorMode = .additive, windowPeriodic: Bool = false
    ) {
        self.nFFT = nFFT
        self.preemph = preemph
        self.nMels = nMels
        self.padTo = max(1, padTo)
        self.winLength = winLength
        var cfg = fa_mel_config(
            sample_rate: Int32(sampleRate), n_mels: Int32(nMels), n_fft: Int32(nFFT), hop_length: Int32(hopLength),
            win_length: Int32(winLength), preemph: preemph, pad_to: Int32(padTo), log_floor: logFloor,
            log_floor_mode: logFloorMode == .additive ? 0 : 1, window_periodic: windowPeriodic ? 1 : 0)
        var h: OpaquePointer?
        let status = fa_mel_create(&cfg, &h)
        precondition(status == FA_STATUS_OK, "fa_mel_create: \(String(cString: fa_last_error()))")
        handle = h
    }

    deinit { fa_mel_destroy(handle) }

    private func run(
        _ audio: UnsafeBufferPointer<Float>, last: Float, mode: Int32, expected: Int?, layout: Int32
    ) -> (mel: [Float], melLength: Int, numFrames: Int) {
        let frames = Int(fa_mel_frame_count(handle, Int64(audio.count), mode, Int64(expected ?? -1)))
        let empty = frames <= 0 || audio.isEmpty
        let padded = empty ? 1 : (mode == 2 ? frames : ((frames + padTo - 1) / padTo) * padTo)
        var out = [Float](repeating: 0, count: nMels * padded)
        var melLength: Int64 = 0
        var numFrames: Int64 = 0
        let status = out.withUnsafeMutableBufferPointer { dst in
            fa_mel_compute(handle, audio.baseAddress, audio.count, last, mode, Int64(expected ?? -1), layout,
                           dst.baseAddress, dst.count, &melLength, &numFrames)
        }
        precondition(status == FA_STATUS_OK, "fa_mel_compute: \(String(cString: fa_last_error()))")
        return (out, Int(melLength), Int(numFrames))
    }

    public func compute(audio: [Float]) -> (mel: [[[Float]]], melLength: Int) {
        let r = audio.withUnsafeBufferPointer { run($0, last: 0, mode: 2, expected: nil, layout: 1) }
        guard r.melLength > 0 else { return ([[[Float]]](), 0) }
        let rows = (0..<nMels).map { m in Array(r.mel[(m * r.melLength)..<((m + 1) * r.melLength)]) }
        return ([rows], r.melLength)
    }

    public func computeFlat(audio: [Float], lastAudioSample: Float = 0) -> (mel: [Float], melLength: Int, numFrames: Int) {
        audio.withUnsafeBufferPointer { run($0, last: lastAudioSample, mode: 0, expected: nil, layout: 1) }
    }

    public func computeFlatTransposed(
        audio: [Float], lastAudioSample: Float = 0, paddingMode: PaddingMode = .center, expectedFrameCount: Int? = nil
    ) -> (mel: [Float], melLength: Int, numFrames: Int) {
        audio.withUnsafeBufferPointer {
            run($0, last: lastAudioSample, mode: paddingMode == .center ? 0 : 1, expected: expectedFrameCount, layout: 0)
        }
    }

    public func getHannWindow() -> [Float] {
        var w = [Float](repeating: 0, count: winLength)
        _ = w.withUnsafeMutableBufferPointer { fa_mel_get_window(handle, $0.baseAddress, $0.count) }
        return w
    }

    public func getFilterbank() -> [[Float]] {
        let bins = nFFT / 2 + 1
        var flat = [Float](repeating: 0, count: nMels * bins)
        _ = flat.withUnsafeMutableBufferPointer { fa_mel_get_filterbank(handle, $0.baseAddress, $0.count) }
        return (0..<nMels).map { Array(flat[($0 * bins)..<(($0 + 1) * bins)]) }
    }
}


// MARK: - Callers directly behind AudioMelSpectrogram, post-processing on the GPU

/// Body of UnifiedMelExtractor.features(window:validCount:) (ASR/Parakeet/Unified/UnifiedMelExtractor.swift:52-86):
/// returns the packed [nMels x totalFrames] floats and the valid frame count; the caller wraps them in MLMultiArrays.
func unifiedMelFeatures(handle: OpaquePointer, window: [Float], validCount: Int, nMels: Int) throws -> (mel: [Float], validFrames: Int32) {
    let totalFrames = window.count / 160 + 1
    var out = [Float](repeating: 0, count: nMels * totalFrames)
    var frames: Int64 = 0
    var valid: Int32 = 0
    let status = fa_mel_unified_features(handle, window, window.count, validCount, &out, out.count, &frames, &valid)
    guard status == FA_STATUS_OK else {
        throw NSError(domain: "fluidaudio_b200", code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
    return (out, valid)
}

/// Replacement for the arithmetic of LSEENDPreprocessor.processAudioQueue (Diarizer/LS-EEND/LSEENDPreprocessor.swift:
/// 249-283); `cmnMean` / `cmnCount` are the preprocessor's own stored properties.
func lseendMelFeatures(handle: OpaquePointer, audioChunk: [Float], nMels: Int, cmnMean: inout [Float], cmnCount: inout Int64) throws -> [Float] {
    let frames = max(0, (audioChunk.count - 512) / 160 + 1)
    var out = [Float](repeating: 0, count: max(frames, 1) * nMels)
    var produced: Int64 = 0
    let status = fa_mel_lseend_features(handle, audioChunk, audioChunk.count, &cmnMean, &cmnCount, &out, out.count, &produced)
    guard status == FA_STATUS_OK else {
        throw NSError(domain: "fluidaudio_b200", code: Int(status.rawValue),
                      userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
    return Array(out.prefix(Int(produced) * nMels))
}
