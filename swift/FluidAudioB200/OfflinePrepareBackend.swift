// The arithmetic of OfflineDiarizerManager.prepare around the two networks, on an sm_90a GPU:
//   OfflineSegmentationBackend    replaces populateWindow and the per-frame decoding loop of OfflineSegmentationProcessor.process
//                                 (Diarizer/Offline/Segmentation/OfflineSegmentationProcessor.swift:118-187, 321-405)
//   OfflineEmbeddingPlanBackend   replaces the chunk loop and processChunk's mask bookkeeping of OfflineEmbeddingExtractor
//                                 (Diarizer/Offline/Extraction/OfflineEmbeddingExtractor.swift:421-707)
//   WeightInterpolationBackend    WeightInterpolation.resample2D (Diarizer/Offline/Extraction/WeightInterpolation.swift:118-136)
// The model predictions stay where they are; these calls take and return flat arrays.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

public enum OfflinePrepareError: Error { case status(fa_status, String) }

private func check(_ status: fa_status) throws {
    guard status == FA_STATUS_OK else { throw OfflinePrepareError.status(status, String(cString: fa_last_error())) }
}

private func segConfig(_ config: OfflineDiarizerConfig) -> fa_seg_config {
    var c = fa_seg_config()
    fa_seg_default_config(&c)
    c.sample_rate = Int32(config.sampleRate)
    c.window_duration = config.windowDuration
    c.step_ratio = config.segmentationStepRatio
    c.speech_onset_threshold = config.speechOnsetThreshold
    return c
}

public struct OfflineSegmentationBackend {
    public let config: OfflineDiarizerConfig
    public init(config: OfflineDiarizerConfig) { self.config = config }

    /// Windows `first ..< first + count` as one [count x samplesPerWindow] array, and their chunkOffsets.
    public func windows(audio: [Float], first: Int, count: Int) throws -> (windows: [Float], chunkOffsets: [Double]) {
        var c = segConfig(config)
        var out = [Float](repeating: 0, count: count * config.samplesPerWindow)
        var offsets = [Double](repeating: 0, count: count)
        try check(fa_seg_windows(audio, Int64(audio.count), &c, Int32(first), Int32(count), &out, &offsets))
        return (out, offsets)
    }

    /// logits [chunks x frames x classes] -> logProbs (same shape), speakerWeights [chunks x frames x 3], class histogram, speech frames.
    public func decode(logits: [Float], chunks: Int, frames: Int, classes: Int) throws
        -> (logProbs: [Float], speakerWeights: [Float], classHistogram: [Int64], speechFrames: Int64)
    {
        var c = segConfig(config)
        var logProbs = [Float](repeating: 0, count: logits.count)
        var weights = [Float](repeating: 0, count: chunks * frames * 3)
        var histogram = [Int64](repeating: 0, count: 8)
        var speech: Int64 = 0
        try check(fa_seg_decode(logits, Int32(chunks), Int32(frames), Int32(classes), &c, &logProbs, &weights, &histogram, &speech))
        return (logProbs, weights, histogram, speech)
    }
}

public struct OfflineEmbeddingPlan {
    public var chunkIndex: [Int32], speakerIndex: [Int32], startFrame: [Int32], endFrame: [Int32]
    public var startTime: [Double], endTime: [Double]
    public var reuseOf: [Int32]            // entry whose embedding this one reuses (maskSimilarity), -1 = its own
    public var frameWeights: [Float]       // [count x frames]        TimedEmbedding.frameWeights
    public var modelWeights: [Float]       // [count x weightFrames]  the embedding model's weights input
    public var count: Int
}

public struct OfflineEmbeddingPlanBackend {
    public let config: OfflineDiarizerConfig
    public let weightFrameCount: Int, audioSampleCount: Int, fbankBatchLimit: Int
    public init(config: OfflineDiarizerConfig, weightFrameCount: Int, audioSampleCount: Int, fbankBatchLimit: Int) {
        self.config = config
        self.weightFrameCount = weightFrameCount
        self.audioSampleCount = audioSampleCount
        self.fbankBatchLimit = fbankBatchLimit
    }

    public func plan(segmentation: SegmentationOutput, totalSamples: Int) throws -> OfflineEmbeddingPlan {
        var seg = segConfig(config)
        var p = fa_embed_plan_config()
        fa_embed_plan_default_config(&p)
        p.exclude_overlap = config.embeddingExcludeOverlap ? 1 : 0
        p.min_segment_duration = config.minSegmentDuration
        if case .maskSimilarity(let threshold) = config.embeddingSkipStrategy { p.skip_threshold = threshold }
        p.weight_frames = Int32(weightFrameCount)
        p.audio_sample_count = Int32(audioSampleCount)
        p.fbank_batch = Int32(fbankBatchLimit)
        let chunks = segmentation.numChunks, frames = segmentation.numFrames, speakers = segmentation.numSpeakers
        let flat = segmentation.speakerWeights.flatMap { $0.flatMap { $0 } }
        let cap = max(1, chunks * speakers)
        var plan = OfflineEmbeddingPlan(
            chunkIndex: .init(repeating: 0, count: cap), speakerIndex: .init(repeating: 0, count: cap),
            startFrame: .init(repeating: 0, count: cap), endFrame: .init(repeating: 0, count: cap),
            startTime: .init(repeating: 0, count: cap), endTime: .init(repeating: 0, count: cap),
            reuseOf: .init(repeating: -1, count: cap), frameWeights: .init(repeating: 0, count: cap * max(1, frames)),
            modelWeights: .init(repeating: 0, count: cap * weightFrameCount), count: 0)
        var n: Int32 = 0
        try check(fa_embedding_plan(
            flat, Int32(chunks), Int32(frames), Int32(speakers), segmentation.chunkOffsets, Int32(segmentation.chunkOffsets.count),
            segmentation.frameDuration, Int64(totalSamples), &seg, &p, &plan.chunkIndex, &plan.speakerIndex, &plan.startFrame,
            &plan.endFrame, &plan.startTime, &plan.endTime, nil, nil, &plan.reuseOf, &plan.frameWeights, &plan.modelWeights, &n, nil))
        plan.count = Int(n)
        return plan
    }

    /// The fbank model's input rows [chunks.count x audioSampleCount] of the listed chunks.
    public func fbankWindows(audio: [Float], chunkOffsets: [Double], chunks: [Int32]) throws -> [Float] {
        var seg = segConfig(config)
        var out = [Float](repeating: 0, count: chunks.count * audioSampleCount)
        try check(fa_embed_windows(audio, Int64(audio.count), chunkOffsets, Int32(chunkOffsets.count), chunks, Int32(chunks.count),
                                   &seg, Int32(audioSampleCount), &out))
        return out
    }
}

public enum WeightInterpolationBackend {
    public static func resample2D(_ rows: [[Float]], to outputLength: Int) throws -> [[Float]] {
        guard let first = rows.first, !first.isEmpty, outputLength > 0 else { return [] }
        var out = [Float](repeating: 0, count: rows.count * outputLength)
        try check(fa_weight_resample(rows.flatMap { $0 }, Int64(rows.count), Int32(first.count), Int32(outputLength), &out))
        return (0..<rows.count).map { Array(out[$0 * outputLength..<($0 + 1) * outputLength]) }
    }
}
