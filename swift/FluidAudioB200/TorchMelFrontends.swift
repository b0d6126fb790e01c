// Drop-ins for the reference's three torch-style log-mel frontends, with their public signatures:
//   CohereMelSpectrogram   Sources/FluidAudio/ASR/Cohere/CoherePipeline.swift:41-324
//   StyleTTS2MelExtractor  Sources/FluidAudio/TTS/StyleTTS2/Pipeline/Preprocess/StyleTTS2MelExtractor.swift
//   LuxTtsMelExtractor     Sources/FluidAudio/TTS/LuxTts/LuxTtsMelExtractor.swift
// All arithmetic happens in libfluidaudio_b200.so on an sm_90a GPU (fa_mel_create_ex + fa_mel_*_features); this file only
// marshals buffers.  `handle` is an ordinary fa_mel handle: batches of prompts go through fa_mel_compute_batch on it.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

private func makeHandle(_ cfg: inout fa_mel_ex_config, _ what: String) -> OpaquePointer? {
    var h: OpaquePointer?
    let status = fa_mel_create_ex(&cfg, &h)
    precondition(status == FA_STATUS_OK, "\(what): \(String(cString: fa_last_error()))")
    return h
}

public final class CohereMelSpectrogram {
    public struct Config: Sendable {
        public let sampleRate: Int
        public let winLength: Int
        public let hopLength: Int
        public let nMels: Int
        public let fMin: Float
        public let fMax: Float
        public let preemph: Float
        public let magPower: Float
        public let logZeroGuard: Float
        public let cmvnEpsilon: Float   // the device epilogue implements the default 1e-5

        public init(
            sampleRate: Int = 16_000, winLength: Int = 400, hopLength: Int = 160, nMels: Int = 128, fMin: Float = 0.0,
            fMax: Float = 8_000.0, preemph: Float = 0.97, magPower: Float = 2.0, logZeroGuard: Float = 5.960_464_5e-08,
            cmvnEpsilon: Float = 1.0e-5
        ) {
            self.sampleRate = sampleRate
            self.winLength = winLength
            self.hopLength = hopLength
            self.nMels = nMels
            self.fMin = fMin
            self.fMax = fMax
            self.preemph = preemph
            self.magPower = magPower
            self.logZeroGuard = logZeroGuard
            self.cmvnEpsilon = cmvnEpsilon
        }
    }

    public struct Output {
        public let mel: [[Float]]  // (nMels, nFrames)
        public let validFrames: Int
    }

    public let config: Config
    public let nFFT: Int
    public private(set) var handle: OpaquePointer?

    public init(config: Config = Config()) {
        precondition(config.cmvnEpsilon == 1.0e-5, "the device CMVN epilogue uses cmvnEpsilon 1e-5")
        self.config = config
        var n = 1
        while n < config.winLength { n <<= 1 }
        self.nFFT = n
        var cfg = fa_mel_ex_config()
        fa_mel_preset_cohere(&cfg)
        cfg.base.sample_rate = Int32(config.sampleRate)
        cfg.base.win_length = Int32(config.winLength)
        cfg.base.hop_length = Int32(config.hopLength)
        cfg.base.n_mels = Int32(config.nMels)
        cfg.base.n_fft = Int32(n)
        cfg.base.preemph = config.preemph
        cfg.base.log_floor = config.logZeroGuard
        cfg.f_min = config.fMin
        cfg.f_max = config.fMax
        cfg.spectrum_power = config.magPower
        handle = makeHandle(&cfg, "fa_mel_create_ex (Cohere)")
    }

    deinit { fa_mel_destroy(handle) }

    public func validFrameCount(forSamples n: Int) -> Int { max(0, n) / config.hopLength }

    /// compute + padOrTruncate in one call (fixedFrames < 0: compute only): ([nMels][width], featureLength).
    public func features(audio: [Float], fixedFrames: Int = 3_500) -> (mel: [[Float]], featureLength: Int) {
        let width = fixedFrames < 0 ? 1 + audio.count / config.hopLength : fixedFrames
        var out = [Float](repeating: 0, count: max(1, config.nMels * width))
        var frames: Int64 = 0
        var valid: Int64 = 0
        let status = audio.withUnsafeBufferPointer { src in
            out.withUnsafeMutableBufferPointer { dst in
                fa_mel_cohere_features(handle, src.baseAddress, src.count, Int64(fixedFrames), dst.baseAddress, dst.count,
                                       &frames, &valid)
            }
        }
        precondition(status == FA_STATUS_OK, "fa_mel_cohere_features: \(String(cString: fa_last_error()))")
        let rows = (0..<config.nMels).map { m in Array(out[(m * width)..<((m + 1) * width)]) }
        return (rows, Int(valid))
    }

    public func compute(audio: [Float]) -> Output {
        let r = features(audio: audio, fixedFrames: -1)
        return Output(mel: r.mel, validFrames: r.featureLength)
    }

    public static func padOrTruncate(
        mel: [[Float]], validFrames: Int, fixedFrames: Int = 3_500
    ) -> (mel: [[Float]], featureLength: Int) {
        guard !mel.isEmpty else { return (mel, 0) }
        let cur = mel[0].count
        if cur == fixedFrames { return (mel, min(validFrames, fixedFrames)) }
        if cur > fixedFrames { return (mel.map { Array($0.prefix(fixedFrames)) }, min(validFrames, fixedFrames)) }
        let pad = [Float](repeating: 0, count: fixedFrames - cur)
        return (mel.map { $0 + pad }, min(validFrames, fixedFrames))
    }
}

public final class StyleTTS2MelExtractor {
    private let nMels: Int
    private let hopLength: Int
    public private(set) var handle: OpaquePointer?

    public init(
        nFFT: Int = 2_048, winLength: Int = 1_200, hopLength: Int = 300, nMels: Int = 80, filterSampleRate: Int = 16_000,
        mean: Float = -4.0, std: Float = 4.0, logEpsilon: Float = 1e-5
    ) {
        self.nMels = nMels
        self.hopLength = hopLength
        var cfg = fa_mel_ex_config()
        fa_mel_preset_styletts2(&cfg)
        cfg.base.n_fft = Int32(nFFT)
        cfg.base.win_length = Int32(winLength)
        cfg.base.hop_length = Int32(hopLength)
        cfg.base.n_mels = Int32(nMels)
        cfg.base.log_floor = logEpsilon
        cfg.filter_sample_rate = Int32(filterSampleRate)
        cfg.log_mean = mean
        cfg.log_std = std
        handle = makeHandle(&cfg, "fa_mel_create_ex (StyleTTS2)")
    }

    deinit { fa_mel_destroy(handle) }

    /// Flat row-major [nMels * nFrames] plus the frame count (1 + n / hop).
    public func compute(audio: [Float]) -> (mel: [Float], frames: Int) {
        let frames = 1 + audio.count / hopLength
        var out = [Float](repeating: 0, count: nMels * frames)
        var got: Int64 = 0
        let status = audio.withUnsafeBufferPointer { src in
            out.withUnsafeMutableBufferPointer { dst in
                fa_mel_styletts2_features(handle, src.baseAddress, src.count, dst.baseAddress, dst.count, &got)
            }
        }
        precondition(status == FA_STATUS_OK, "fa_mel_styletts2_features: \(String(cString: fa_last_error()))")
        return (out, Int(got))
    }
}

public final class LuxTtsMelExtractor {
    private let hop = 256
    private let nMels = 100
    public private(set) var handle: OpaquePointer?

    public init() {
        var cfg = fa_mel_ex_config()
        fa_mel_preset_luxtts(&cfg)
        handle = makeHandle(&cfg, "fa_mel_create_ex (LuxTTS)")
    }

    deinit { fa_mel_destroy(handle) }

    /// lhotse `compute_num_frames`: `(num_samples + hop/2) / hop`.
    public func frameCount(sampleCount: Int) -> Int { (sampleCount + hop / 2) / hop }

    /// `[T][nMels]` log-mel frames, `T = frameCount(sampleCount:)` (none for empty audio).
    public func extract(audio: [Float]) -> [[Float]] {
        let target = audio.isEmpty ? 0 : frameCount(sampleCount: audio.count)
        guard target > 0 else { return [] }
        var out = [Float](repeating: 0, count: target * nMels)
        var got: Int64 = 0
        let status = audio.withUnsafeBufferPointer { src in
            out.withUnsafeMutableBufferPointer { dst in
                fa_mel_luxtts_features(handle, src.baseAddress, src.count, dst.baseAddress, dst.count, &got)
            }
        }
        precondition(status == FA_STATUS_OK, "fa_mel_luxtts_features: \(String(cString: fa_last_error()))")
        return (0..<Int(got)).map { t in Array(out[(t * nMels)..<((t + 1) * nMels)]) }
    }
}
