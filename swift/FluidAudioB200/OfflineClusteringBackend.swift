// Drop-in for the clustering phase of OfflineDiarizerManager.cluster(_:)
// (Sources/FluidAudio/Diarizer/Offline/Core/OfflineDiarizerManager.swift:286-375): Float->Double, NaN filter, AHC,
// VBx, centroids, argmax assignment — one call into libfluidaudio_b200.so.  AHCClustering / VBxClustering keep their
// own Swift signatures (AHCClustering.swift:20-23, VBxClustering.swift:41-44) and forward to fa_ahc_cluster / fa_vbx_refine.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
import CFluidAudioB200
import Foundation

struct AHCClustering {
    func cluster(embeddingFeatures: [[Double]], threshold: Double) -> [Int] {
        let count = embeddingFeatures.count
        guard count > 0 else { return [] }
        guard let dimension = embeddingFeatures.first?.count, dimension > 0 else { return Array(repeating: 0, count: count) }
        if count == 1 { return [0] }
        let flat = embeddingFeatures.flatMap { $0 }
        var labels = [Int32](repeating: 0, count: count)
        let status = fa_ahc_cluster(flat, count, dimension, threshold, &labels)
        guard status == FA_STATUS_OK else { return Array(0..<count) }   // same fallback as AHCClustering.swift:52-55
        return labels.map(Int.init)
    }
}

struct OfflineClusteringBackend {
    struct Output {
        let assignments: [Int]          // one cluster per embedding (assignEmbeddings)
        let initialClusters: [Int]      // AHC labels of the training rows, -1 for NaN-filtered rows
        let centroids: [[Double]]
        let info: fa_cluster_info
    }

    var threshold: Double = 0.6          // OfflineDiarizerConfig.clusteringThreshold
    var warmStartFa: Double = 0.07
    var warmStartFb: Double = 0.8
    var maxIterations: Int = 20
    var convergenceTolerance: Double = 1e-4
    // OfflineDiarizerConfig.Clustering speaker-count constraints; nil -> FA_NO_VALUE.  When they bind, the library
    // re-clusters with K-Means exactly like VBxClustering.refineWithConstraints (VBxClustering.swift:685-733).
    var numSpeakers: Int? = nil
    var minSpeakers: Int? = nil
    var maxSpeakers: Int? = nil
    /// TimedEmbedding.chunkIndex per embedding: switches on the reference's default constrained assignment
    /// (ConstrainedClusterAssignment.swift:20-42) through fa_diarize_cluster_chunks.
    var chunkIndices: [Int32]? = nil

    /// `embedding256`: N x dim row-major Float (TimedEmbedding.embedding256), `rho128`: N x rhoDim row-major Double,
    /// `psi`: PLDATransform.phiParameters.
    func cluster(embedding256: [Float], rho128: [Double], count: Int, dim: Int, rhoDim: Int, psi: [Double]) throws -> Output {
        var cfg = fa_cluster_config()
        fa_cluster_default_config(&cfg)
        cfg.threshold = threshold
        cfg.vbx.Fa = warmStartFa
        cfg.vbx.Fb = warmStartFb
        cfg.vbx.max_iterations = Int32(maxIterations)
        cfg.vbx.epsilon = convergenceTolerance
        cfg.num_speakers = numSpeakers.map(Int32.init) ?? FA_NO_VALUE
        cfg.min_speakers = minSpeakers.map(Int32.init) ?? FA_NO_VALUE
        cfg.max_speakers = maxSpeakers.map(Int32.init) ?? FA_NO_VALUE
        var labels = [Int32](repeating: 0, count: count)
        var initial = [Int32](repeating: 0, count: count)
        let maxCentroids = 64
        var centroids = [Double](repeating: 0, count: maxCentroids * dim)
        var info = fa_cluster_info()
        let status: fa_status
        if let chunks = chunkIndices {
            status = fa_diarize_cluster_chunks(embedding256, rho128, count, dim, rhoDim, psi, &cfg, chunks, &labels,
                                               &initial, &centroids, Int32(maxCentroids), &info)
        } else {
            status = fa_diarize_cluster(embedding256, rho128, count, dim, rhoDim, psi, &cfg, &labels, &initial,
                                        &centroids, Int32(maxCentroids), &info)
        }
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fluidaudio_b200", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        let k = min(Int(info.centroid_count), maxCentroids)
        return Output(
            assignments: labels.map(Int.init), initialClusters: initial.map(Int.init),
            centroids: (0..<k).map { Array(centroids[($0 * dim)..<(($0 + 1) * dim)]) }, info: info)
    }

    /// Many meetings on one GPU (several side by side on disjoint SM partitions): meeting m is rows
    /// `setOffsets[m] ..< setOffsets[m + 1]` of the packed arrays.  `chunkIndices` (numbered inside each meeting) selects
    /// the reference's default constrained assignment per meeting (fa_diarize_cluster_batch_chunks), nil the plain argmax.
    func clusterBatch(embedding256: [Float], rho128: [Double], setOffsets: [Int64], dim: Int, rhoDim: Int,
                      psi: [Double]) throws -> (assignments: [Int32], info: [fa_cluster_info]) {
        var cfg = fa_cluster_config()
        fa_cluster_default_config(&cfg)
        cfg.threshold = threshold
        cfg.vbx.Fa = warmStartFa
        cfg.vbx.Fb = warmStartFb
        cfg.vbx.max_iterations = Int32(maxIterations)
        cfg.vbx.epsilon = convergenceTolerance
        cfg.num_speakers = numSpeakers.map(Int32.init) ?? FA_NO_VALUE
        cfg.min_speakers = minSpeakers.map(Int32.init) ?? FA_NO_VALUE
        cfg.max_speakers = maxSpeakers.map(Int32.init) ?? FA_NO_VALUE
        let sets = max(setOffsets.count - 1, 0)
        var labels = [Int32](repeating: 0, count: Int(setOffsets.last ?? 0))
        var infos = [fa_cluster_info](repeating: fa_cluster_info(), count: max(sets, 1))
        let status: fa_status
        if let chunks = chunkIndices {
            status = fa_diarize_cluster_batch_chunks(embedding256, rho128, setOffsets, Int32(sets), dim, rhoDim, psi, &cfg,
                                                     chunks, &labels, &infos)
        } else {
            status = fa_diarize_cluster_batch(embedding256, rho128, setOffsets, Int32(sets), dim, rhoDim, psi, &cfg,
                                              &labels, &infos)
        }
        guard status == FA_STATUS_OK else {
            throw NSError(domain: "fluidaudio_b200", code: Int(status.rawValue),
                          userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
        }
        return (labels, Array(infos.prefix(sets)))
    }
}


/// Reads the JSON that OfflineDiarizerManager.exportEmbeddings writes (OfflineDiarizerManager.swift:913-955) — the
/// wire format between a Mac running the CoreML models and the GPU clustering backend.
struct EmbeddingExportFile {
    var chunkIndex: [Int32] = [], speakerIndex: [Int32] = [], startFrame: [Int32] = [], endFrame: [Int32] = []
    var startTime: [Double] = [], endTime: [Double] = [], embedding256: [Float] = [], rho128: [Double] = []
    var cluster: [Int32] = []
    var count = 0, embeddingDim = 0, rhoDim = 0

    init(path: String) throws {
        var n = 0, e = 0, r = 0
        var status = fa_export_shape(path, &n, &e, &r)
        guard status == FA_STATUS_OK else { throw EmbeddingExportFile.error(status) }
        count = n; embeddingDim = e; rhoDim = r
        chunkIndex = .init(repeating: 0, count: n); speakerIndex = chunkIndex; startFrame = chunkIndex
        endFrame = chunkIndex; cluster = chunkIndex
        startTime = .init(repeating: 0, count: n); endTime = startTime
        embedding256 = .init(repeating: 0, count: n * e); rho128 = .init(repeating: 0, count: n * r)
        status = fa_export_read(path, n, e, r, &chunkIndex, &speakerIndex, &startFrame, &endFrame, &startTime, &endTime,
                                &embedding256, &rho128, &cluster)
        guard status == FA_STATUS_OK else { throw EmbeddingExportFile.error(status) }
    }

    private static func error(_ status: fa_status) -> NSError {
        NSError(domain: "fluidaudio_b200", code: Int(status.rawValue),
                userInfo: [NSLocalizedDescriptionKey: String(cString: fa_last_error())])
    }
}
