// Drop-in for the conversion core of Sources/FluidAudio/Shared/AudioConverter.swift (same public surface for the
// array / buffer entry points: resample(_:from:) :60-71, resampleBuffer(_:) :77-85).  Mixdown, int16 widening and the
// sample-rate conversion run on an sm_90a GPU behind fa_audio_resample; file decoding (AVAudioFile, :91-130) and
// CMSampleBuffer handling (:134-297) stay where they are and hand their PCM to `resampleBuffer`.
// One or two channels: the library's documented Kaiser-windowed-sinc filter replaces Apple's closed AVAudioConverter
// ("parity unpinned" for sample values; the output length follows Int(n / ratio), inside the reference tests' 1 %).
// More than two channels: AudioConverter.linearResample (:388-442), bit for bit.
// NOT compiled in this repository (no Swift toolchain in the build image) — see INTEGRATION.md.
@preconcurrency import AVFoundation
import CFluidAudioB200
import Foundation

final public class AudioConverter: Sendable {
    private let targetRate: Double

    public init(sampleRate: Double = 16000) { targetRate = sampleRate }

    public func resample(_ samples: [Float], from inputRate: Double) throws -> [Float] {
        guard !samples.isEmpty else { return [] }
        if inputRate == targetRate { return samples }                       // :66-68
        return try convert(samples, frames: samples.count, rate: inputRate, channels: 1, format: FA_PCM_F32, interleaved: false)
    }

    public func resampleBuffer(_ buffer: AVAudioPCMBuffer) throws -> [Float] {
        let fmt = buffer.format
        let frames = Int(buffer.frameLength)
        let channels = Int(fmt.channelCount)
        if let f = buffer.floatChannelData {
            if fmt.isInterleaved {
                return try convert(UnsafeBufferPointer(start: f[0], count: frames * channels), frames: frames,
                                   rate: fmt.sampleRate, channels: channels, format: FA_PCM_F32, interleaved: true)
            }
            var planar = [Float](repeating: 0, count: frames * channels)    // floatChannelData: one pointer per channel
            for c in 0..<channels { planar.replaceSubrange(c * frames..<(c + 1) * frames, with: UnsafeBufferPointer(start: f[c], count: frames)) }
            return try convert(planar, frames: frames, rate: fmt.sampleRate, channels: channels, format: FA_PCM_F32, interleaved: false)
        }
        if let i = buffer.int16ChannelData, fmt.isInterleaved || channels == 1 {
            return try convert(UnsafeBufferPointer(start: i[0], count: frames * channels), frames: frames,
                               rate: fmt.sampleRate, channels: channels, format: FA_PCM_I16, interleaved: true)
        }
        throw AudioConverterError.failedToCreateBuffer
    }

    private func convert<C: Collection>(_ pcm: C, frames: Int, rate: Double, channels: Int, format: Int32, interleaved: Bool)
        throws -> [Float]
    {
        var f = fa_audio_format(in_rate: rate, out_rate: targetRate, channels: Int32(channels), format: format,
                                interleaved: interleaved ? 1 : 0, algorithm: Int32(FA_RESAMPLE_AUTO))
        let count = Int(fa_resample_output_count(&f, Int64(frames)))
        var out = [Float](repeating: 0, count: max(count, 0))
        var produced: Int64 = 0
        let status = pcm.withContiguousStorageIfAvailable { p in
            fa_audio_resample(p.baseAddress, Int64(frames), &f, &out, Int64(out.count), &produced)
        }
        guard status == FA_STATUS_OK else { throw AudioConverterError.conversionFailed(nil) }
        return out
    }
}

// AudioMelSpectrogram + AudioConverter fused (no reference counterpart: the two calls back to back, minus the PCIe trip
// of the converted samples):  let (mel, len, frames) = mel.computeFlatTransposed(pcm16: samples, sampleRate: 44100, channels: 2)
extension AudioMelSpectrogram {
    public func computeFlatTransposed(pcm16: [Int16], sampleRate: Double, channels: Int) -> (mel: [Float], melLength: Int, numFrames: Int) {
        var f = fa_audio_format(in_rate: sampleRate, out_rate: 16000, channels: Int32(channels), format: Int32(FA_PCM_I16),
                                interleaved: 1, algorithm: Int32(FA_RESAMPLE_AUTO))
        let frames = pcm16.count / max(channels, 1)
        let n = Int(fa_resample_output_count(&f, Int64(frames)))
        let cap = Int(fa_mel_frame_count(rawHandle, Int64(n), 0, -1)) * melBins
        var out = [Float](repeating: 0, count: max(cap, melBins))
        var ml: Int64 = 0, nf: Int64 = 0, rs: Int64 = 0
        _ = fa_audio_to_mel(rawHandle, pcm16, Int64(frames), &f, 0, 0, 0, &out, out.count, &ml, &nf, &rs)
        return (Array(out.prefix(Int(nf) * melBins)), Int(ml), Int(nf))
    }
}
