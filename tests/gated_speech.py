"""Signals whose silence-gate mask is known -- TEST INFRASTRUCTURE (plain numpy, seeded, no GPU).

The gate (oracle.pipeline.effective_mask, csrc/features.cu k_frame_mse + k_gate) keeps the frames whose mean square lies within
`threshold_db` of the loudest frame of the window.  synthetic.synthetic_speech's own gaps still carry noise 40 dB under the speech, so
at the usual threshold of 60 every frame of it is effective.  Here continuous speech (silence_fraction=0) is multiplied by a gate of
the test's own: 1 on the loud part, FLOOR_DB (or exactly 0) on the quiet part.

  * window_with_count: one convert window with exactly `target` effective frames, the loud part laid out as 'head', 'tail' or 'comb';
    the loud length is found by bisection on the oracle's mask and the result is asserted.
  * peak_window: one window and the threshold at which exactly its loudest frame is effective.  A frame is fft_length = 1024 samples
    wide and frames are hop = 120 apart, so every sample lies in 8 or 9 frames and the neighbours of the loudest frame share 904 of its
    samples: no signal has fewer than a handful of effective frames at 60 dB.  One effective frame needs a threshold of a fraction of
    a dB, taken here from the two loudest frames of plain speech.
  * stream_with_pauses: a stream whose pauses last from 0.1 s to longer than the convert window; step_counts gives the oracle's
    effective frames of every session step.
  * mask_margin: the distance of the closest frame from the threshold, in dB.  The device and numpy both evaluate log10 in FP64 but
    not necessarily to the same last bit: a case is only used when its margin is at least MIN_MARGIN_DB.
"""
import numpy as np

from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import synthetic

CFG = opipe.PathConfig()
FS, HOP = CFG.fs, CFG.hop
FLOOR_DB = -68.0              # quiet part under the loud part: gated at 60 dB; with the speech's own 10 dB of level changes, effective at 80
MIN_MARGIN_DB = 1e-6
# 'comb': the window is cut into segments of these relative widths and the first part of each is loud, so the loud runs and the gaps
# between them all differ in length and an effective frame's rank falls behind its index by a different amount after every gap
COMB_SEGMENTS = (0.13, 0.31, 0.19, 0.37)
PATTERNS = ('head', 'tail', 'comb')
# (pattern, effective frames at 60 dB, quiet part digital zeros) of the window cases: one frame each side of the padded lengths 128 and
# 256.  From 255 frames on at most one gap of a comb is still wide enough to gate a frame, so 'comb' stops at 129
WINDOW_CASES = ([(p, t, False) for t in (127, 128, 129) for p in PATTERNS] + [(p, t, False) for t in (255, 256, 257) for p in ('head', 'tail')]
                + [('comb', 128, True), ('tail', 256, True)])


def frame_db(wave, n_frames):
    """dB of every frame under the loudest, as effective_mask computes it."""
    mse = oworld.frame_mse(np.asarray(wave), CFG.fft_length, HOP, n_frames)
    ref = 10.0 * np.log10(max(1e-10, float(mse.max())))
    return 10.0 * np.log10(np.maximum(1e-10, mse)) - ref


def mask_margin(wave, n_frames, thr):
    """smallest |db + thr| over the frames: how far the closest decision is from flipping (inf without a gate)"""
    if thr is None or n_frames == 0:
        return float('inf')
    return float(np.abs(frame_db(wave, n_frames) + thr).min())


def count_effective(wave, n_frames, thr):
    return int(opipe.effective_mask(np.asarray(wave), n_frames, CFG, thr).sum())


def _speech(n, stream):
    return synthetic.synthetic_speech(n / FS, stream=stream, silence_fraction=0.0)[:n].astype(np.float64)


def _loud(n, loud_samples, pattern):
    """bool[n]: the loud samples; the sets grow with loud_samples (nested), so the effective count grows with it"""
    loud = np.zeros(n, bool)
    if pattern == 'head':
        loud[:loud_samples] = True
    elif pattern == 'tail':
        loud[n - loud_samples:] = True
    elif pattern == 'comb':
        edges = np.round(np.concatenate([[0.0], np.cumsum(COMB_SEGMENTS)]) / sum(COMB_SEGMENTS) * n).astype(int)
        for a, b in zip(edges[:-1], edges[1:]):
            loud[a:a + (b - a) * loud_samples // n] = True
    else:
        raise ValueError(pattern)
    return loud


def _gated(x, loud, zeros):
    quiet = 0.0 if zeros else 10.0 ** (FLOOR_DB / 20.0)
    return (x * np.where(loud, 1.0, quiet)).astype(np.float32)


def window_with_count(target, Tw=260, thr=60.0, pattern='head', zeros=False, stream=700):
    """(wave of Tw * hop samples, oracle mask) with exactly `target` effective frames at `thr`."""
    n = Tw * HOP
    x = _speech(n, stream)
    lo, hi = 0, n                                   # smallest loud length whose count reaches the target
    while lo < hi:
        mid = (lo + hi) // 2
        if count_effective(_gated(x, _loud(n, mid, pattern), zeros), Tw, thr) >= target:
            hi = mid
        else:
            lo = mid + 1
    wave = _gated(x, _loud(n, lo, pattern), zeros)
    mask = opipe.effective_mask(wave, Tw, CFG, thr)
    assert int(mask.sum()) == target, (pattern, target, int(mask.sum()), lo)
    assert mask_margin(wave, Tw, thr) >= MIN_MARGIN_DB, (pattern, target, mask_margin(wave, Tw, thr))
    return wave, mask


def peak_window(Tw=260, stream=700):
    """(wave, thr, mask): plain continuous speech and the threshold half way between its two loudest frames."""
    wave = _speech(Tw * HOP, stream).astype(np.float32)
    db = np.sort(frame_db(wave, Tw))
    thr = float(-(db[-1] + db[-2]) / 2.0)
    mask = opipe.effective_mask(wave, Tw, CFG, thr)
    assert int(mask.sum()) == 1 and thr > 0 and mask_margin(wave, Tw, thr) >= MIN_MARGIN_DB, (thr, int(mask.sum()))
    return wave, thr, mask


# (speech seconds, pause seconds), in order.  With 0.3 s chunks and a 1.3 s convert window: the pauses of 0.1 and 0.3 s leave the
# window almost full, those of 0.7 to 1.2 s take it down to under 128 frames, and during the 1.6 s pause one window is quiet from end
# to end -- and then wholly effective again, since the gate is relative to the window's own loudest frame.
PAUSES = ((1.5, 0.1), (0.7, 0.3), (0.5, 0.9), (0.4, 1.6), (0.9, 0.7), (0.3, 1.2), (1.3, 0.0))


def stream_with_pauses(seconds=10.5, stream=710, zeros=False):
    """float32 stream: continuous speech with the pauses of PAUSES (repeated if `seconds` is longer)."""
    n = int(round(seconds * FS))
    x = _speech(n, stream)
    loud = np.zeros(n, bool)
    t = 0
    while t < n:
        for speech, pause in PAUSES:
            loud[t:t + int(round(speech * FS))] = True
            t += int(round((speech + pause) * FS))
    return _gated(x, loud, zeros)


def step_windows(wave, steps, buffer_time=0.3, convert_extra=0.5):
    """The wave window the silence gate of session step k sees (no encode overlap): the samples of frames
    [k * n_feat - 2 * e_conv, (k + 1) * n_feat) of the stream, zeros before its start.  -> list of (Tw * hop,) arrays"""
    rate = FS // HOP
    n_feat, e_conv = round(buffer_time * rate), round(convert_extra * rate)
    Tw = n_feat + 2 * e_conv
    out = []
    for k in range(steps):
        first, w = (k * n_feat - 2 * e_conv) * HOP, np.zeros(Tw * HOP, np.float32)
        lo = max(first, 0)
        w[lo - first:] = wave[lo:first + Tw * HOP]
        out.append(w)
    return out


def step_counts(wave, steps, thr, buffer_time=0.3, convert_extra=0.5):
    """[(effective frames, stage-1 bucket = padded length / 128, margin dB)] per session step, from the oracle's masks"""
    rows = []
    for w in step_windows(wave, steps, buffer_time, convert_extra):
        Tw = len(w) // HOP
        c = count_effective(w, Tw, thr)
        rows.append((c, (c + 128 - c % 128) // 128 if c else 0, mask_margin(w, Tw, thr)))
    return rows
