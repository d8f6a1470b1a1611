"""FP64 numpy restatement of the pitch correction (DESIGN.md §4m, DECIDE P1-P4; csrc/pitch.cu) -- TEST INFRASTRUCTURE.

  * PitchStream: the streaming correction; push(f0) corrects the frames in stream order and carries c, n_prev and voiced_prev to the
    next push, so pushes of any length give the whole signal's values.  set() changes the settings from the next push on.
  * pitch_correct: the whole signal from a fresh state (ryk_pitch_correct).
The device computes log2 and exp2 with its own libm, so it agrees with this oracle to ~1e-15 relative, not bit for bit; a note choice can
differ only where s lies within rounding of a decision boundary (boundary_distance).
"""
import math

import numpy as np

HOLD = 0.5 + 0.15            # P1: hysteresis, semitones
NO_NOTE = -(1 << 28)
SCALES = {'chromatic': 0xfff, 'major': 0b101010110101, 'minor': 0b010110101101}
NOTE_NAMES = ('C', 'C#', 'D', 'D#', 'E', 'F', 'F#', 'G', 'G#', 'A', 'A#', 'B')


def in_scale(n, key, scale):
    return (scale >> ((n - key) % 12)) & 1


def beta(hop_ms, retune_ms):
    return 1.0 if retune_ms == 0 else -math.expm1(-hop_ms / retune_ms)


def voiced(f0):
    f0 = np.asarray(f0, np.float64)
    return (f0 > 0) & (f0 < np.inf)


def semitones(f0, a4=440.0):
    """s = 69 + 12 (log2 f0 - log2 a4) of every frame (NaN where unvoiced): finite for every positive finite f0"""
    f0 = np.asarray(f0, np.float64)
    v = voiced(f0)
    s = np.full(len(f0), np.nan)
    s[v] = 69.0 + 12.0 * (np.log2(f0[v]) - math.log2(a4))
    return s


def nearest(s, key, scale):
    """the nearest scale note to s, ties to the lower"""
    lo = math.floor(s)
    best, bd = lo, math.inf
    for k in range(lo - 6, lo + 8):
        if in_scale(k, key, scale):
            d = abs(s - k)
            if d < bd:
                best, bd = k, d
    return best


def note_hz(n, a4=440.0):
    return a4 * 2.0 ** ((n - 69) / 12.0)


class PitchStream:
    def __init__(self, hop_ms, key=0, scale=0xfff, a4=440.0, retune_ms=50.0, amount=1.0):
        self.hop_ms = hop_ms
        self.set(key, scale, a4, retune_ms, amount)
        self.c, self.n_prev, self.voiced_prev = 0.0, NO_NOTE, 0
        self.meter = (0, 0.0, 0.0)           # (voiced frames, mean cents, max cents) of the last push

    def set(self, key, scale, a4=440.0, retune_ms=50.0, amount=1.0):
        self.key, self.scale, self.a4, self.retune_ms, self.amount = int(key), int(scale), float(a4), float(retune_ms), float(amount)
        self.beta = beta(self.hop_ms, self.retune_ms)

    def push(self, f0, notes=None):
        """corrected f0 (float64) of the frames in stream order; `notes` (a list) receives each voiced frame's target and s"""
        f0 = np.asarray(f0, np.float64)
        out = f0.copy()
        s_all = semitones(f0, self.a4)
        n_voiced, total, mx = 0, 0.0, 0.0
        for i in range(len(f0)):
            if not (f0[i] > 0 and f0[i] < np.inf):
                self.voiced_prev = 0
                continue
            s = float(s_all[i])
            n = nearest(s, self.key, self.scale)
            if in_scale(self.n_prev, self.key, self.scale) and abs(s - self.n_prev) < HOLD:
                n = self.n_prev
            d = float(n) - s
            self.c = self.c + self.beta * (d - self.c) if self.voiced_prev else d
            self.n_prev, self.voiced_prev = n, 1
            out[i] = f0[i] * np.exp2(self.amount * self.c / 12.0)
            cents = abs(self.amount * self.c) * 100.0
            n_voiced += 1
            total += cents
            mx = max(mx, cents)
            if notes is not None:
                notes.append((i, n, s))
        self.meter = (n_voiced, total / n_voiced if n_voiced else 0.0, mx)
        return out


def pitch_correct(f0, hop_ms, key=0, scale=0xfff, a4=440.0, retune_ms=50.0, amount=1.0, notes=None):
    return PitchStream(hop_ms, key, scale, a4, retune_ms, amount).push(f0, notes)


def boundary_distance(s, key, scale, n_prev):
    """how far s lies from the nearest point where the P1 decision could change: a midpoint between two scale notes or the
    hysteresis edge n_prev +- HOLD"""
    best = math.inf
    lo = math.floor(s)
    notes = [k for k in range(lo - 8, lo + 10) if in_scale(k, key, scale)]
    for a, b in zip(notes[:-1], notes[1:]):
        best = min(best, abs(s - (a + b) / 2.0))
    if in_scale(n_prev, key, scale):
        best = min(best, abs(abs(s - n_prev) - HOLD))
    return best
