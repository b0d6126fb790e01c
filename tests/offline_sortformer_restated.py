"""A literal pure-Python restatement of OfflineSortformerDiarizer's window work (test infrastructure): processComplete's
window loop (OfflineSortformerDiarizer.swift:279-363), runOffline's copy (:98-119) and SortformerSpeakerStitcher
.alignment with its swap recursion (SortformerSpeakerStitcher.swift:27-90), in float32 numpy scalars, so every product
and sum rounds once as Swift's Float does.  It shares no code with the oracle or the library."""
import numpy as np

WINDOW_OUT, SUBSAMPLING, SPEAKERS, MELS = 384, 8, 4, 128
WINDOW_MEL = WINDOW_OUT * SUBSAMPLING
F32_MAX = np.float32(np.finfo(np.float32).max)


def frame_duration_seconds():
    """Float(subsamplingFactor) * Float(melStride) / Float(sampleRate)"""
    return np.float32(np.float32(np.float32(8) * np.float32(160)) / np.float32(16000))


def clamp_overlap(overlap):
    return max(0, min(int(overlap), WINDOW_OUT - 1))


def plan(num_mel_frames, overlap):
    """(windows, totalOut) by running the loop"""
    n = int(num_mel_frames)
    if n <= 0:
        return 0, 0
    hop_mel = (WINDOW_OUT - clamp_overlap(overlap)) * SUBSAMPLING
    mel_start, windows = 0, 0
    while mel_start < n:
        valid_mel = min(WINDOW_MEL, n - mel_start)
        windows += 1
        if valid_mel < WINDOW_MEL:
            break
        mel_start += hop_mel
    return windows, (n + SUBSAMPLING - 1) // SUBSAMPLING


def run_offline(mel_time_major, valid_mel_frames):
    frames = min(int(valid_mel_frames), WINDOW_MEL)
    src = np.asarray(mel_time_major, np.float32).reshape(-1)
    dst = np.zeros((MELS, WINDOW_MEL), np.float32)
    dst[:, :frames] = src[:frames * MELS].reshape(frames, MELS).T   # dst[c, t] = src[t * MELS + c]
    return dst, frames


def permutations(n=SPEAKERS):
    """permute(_:_:_:)'s order"""
    array, out = list(range(n)), []

    def rec(k):
        if k == n:
            out.append(list(array))
            return
        for i in range(k, n):
            array[k], array[i] = array[i], array[k]
            rec(k + 1)
            array[k], array[i] = array[i], array[k]

    rec(0)
    return out


def alignment(global_rows, window_rows, frames, num_speakers=SPEAKERS):
    identity = list(range(num_speakers))
    g = np.asarray(global_rows, np.float32).reshape(-1)
    w = np.asarray(window_rows, np.float32).reshape(-1)
    if not (frames > 0 and num_speakers > 0 and g.size >= frames * num_speakers and w.size >= frames * num_speakers):
        return identity
    corr = [[np.float32(0)] * num_speakers for _ in range(num_speakers)]
    with np.errstate(all="ignore"):
        for f in range(frames):
            base = f * num_speakers
            for gi in range(num_speakers):
                gv = g[base + gi]
                if not gv != 0:
                    continue
                for wi in range(num_speakers):
                    corr[gi][wi] = np.float32(corr[gi][wi] + np.float32(gv * w[base + wi]))
        best_perm, best_score = identity, -F32_MAX
        for cand in permutations(num_speakers):
            score = np.float32(0)
            for gi in range(num_speakers):
                score = np.float32(score + corr[gi][cand[gi]])
            if score > best_score:
                best_score, best_perm = score, cand
    mapping = list(identity)
    for gi in range(num_speakers):
        mapping[best_perm[gi]] = gi
    return mapping


def stitch(mel_time_major, num_mel_frames, overlap, model):
    """(global [totalOut x 4], mappings [windows x 4]) with model(mel [128 x 3072], mel_length) -> [384 x 4]"""
    n = int(num_mel_frames)
    if n <= 0:
        return np.zeros((0, SPEAKERS), np.float32), np.zeros((0, SPEAKERS), np.int32)
    rows = np.asarray(mel_time_major, np.float32).reshape(-1)
    overlap_out = clamp_overlap(overlap)
    hop_mel = (WINDOW_OUT - overlap_out) * SUBSAMPLING
    total = (n + SUBSAMPLING - 1) // SUBSAMPLING
    glob = np.zeros(total * SPEAKERS, np.float32)
    filled = [False] * total
    mel_start, window_index, maps = 0, 0, []
    while mel_start < n:
        valid_mel = min(WINDOW_MEL, n - mel_start)
        mel, ml = run_offline(rows[mel_start * MELS:(mel_start + valid_mel) * MELS], valid_mel)
        preds = np.asarray(model(mel, ml), np.float32).reshape(-1)
        valid_out = min(WINDOW_OUT, (valid_mel + SUBSAMPLING - 1) // SUBSAMPLING)
        g_start = mel_start // SUBSAMPLING
        mapping = list(range(SPEAKERS))
        if window_index > 0 and overlap_out > 0:
            ov = min(overlap_out, valid_out, max(0, total - g_start))
            if ov > 0:
                mapping = alignment(glob[g_start * SPEAKERS:(g_start + ov) * SPEAKERS], preds[:ov * SPEAKERS], ov)
        maps.append(mapping)
        with np.errstate(all="ignore"):
            for j in range(valid_out):
                gf = g_start + j
                if not gf < total:
                    break
                for w in range(SPEAKERS):
                    idx = gf * SPEAKERS + mapping[w]
                    if filled[gf]:
                        glob[idx] = np.float32(np.float32(glob[idx] + preds[j * SPEAKERS + w]) * np.float32(0.5))
                    else:
                        glob[idx] = preds[j * SPEAKERS + w]
                filled[gf] = True
        window_index += 1
        if valid_mel < WINDOW_MEL:
            break
        mel_start += hop_mel
    return glob.reshape(total, SPEAKERS), np.array(maps, np.int32).reshape(-1, SPEAKERS)
