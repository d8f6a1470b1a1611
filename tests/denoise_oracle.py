"""FP64 numpy reference of the input noise suppression (DESIGN.md DECIDE N1-N3) for the tests.

DenoiseOracle is the streaming filter a session runs: push() takes the model-rate chunk of a step and returns the filtered chunk of
concat(zeros(D), z); the settings a test changes between pushes apply from the next push, as the session's setters apply from the next
submitted step.  denoise() is the whole-signal call (ryk_denoise).  Both sum every output sample over its frames in ascending frame order
from 0.0, so a chunked stream equals the whole signal exactly."""
from typing import Optional

import numpy as np

N, H = 512, 128                  # frame length and hop (N1)
NB = N // 2 + 1                  # rfft bins
D = N - 1                        # the session's delay (N3)
ALPHA = 0.98                     # decision-directed smoothing (N2)
WINDOW = np.sqrt(0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(N) / N))     # periodic sqrt-Hann


def gain_floor(reduction_db: float) -> float:
    return 10.0 ** (-float(reduction_db) / 20.0)


def frame_spectrum(x: np.ndarray, m: int) -> np.ndarray:
    """X_m = rfft(w * x[s_m : s_m + N]), s_m = m H - (N - H), x zero before 0 and after its end"""
    s = m * H - (N - H)
    seg = np.zeros(N)
    lo, hi = max(s, 0), min(s + N, len(x))
    if hi > lo:
        seg[lo - s:hi - s] = x[lo:hi]
    return np.fft.rfft(WINDOW * seg)


def frame_powers(x, first: int, count: int) -> np.ndarray:
    """(count, NB) P_m = |X_m|^2 of frames first .. first + count - 1"""
    x = np.asarray(x, np.float64)
    out = []
    for m in range(first, first + count):
        X = frame_spectrum(x, m)
        out.append(X.real * X.real + X.imag * X.imag)
    return np.array(out)


class DenoiseOracle:
    """The session's filter, step by step.  Frame m is processed in the push whose samples hold its last sample m H + H - 1."""

    def __init__(self, reduction_db: float = 20.0, phi: Optional[np.ndarray] = None):
        self.g = gain_floor(reduction_db)
        self.phi = np.zeros(NB) if phi is None else np.array(phi, np.float64)
        self.x = np.zeros(0)
        self.acc = np.zeros(D)                   # FP64 sums of samples -D .. len(x) + N - (N - H) - 1, index t + D
        self.G, self.Pp = np.ones(NB), np.zeros(NB)
        self.frames_done = 0
        self.learn_left, self.learn_total, self.learn_sum = 0, 0, np.zeros(NB)
        self._reduction, self._profile, self._learn = None, None, None

    # ---- settings: from the next push on ----
    def set_reduction(self, reduction_db: float):
        self._reduction = float(reduction_db)

    def set_profile(self, phi):
        self._profile = np.array(phi, np.float64)
        self._learn = 0                           # cancels a learning in progress

    def learn(self, n_frames: int):
        self._learn = int(n_frames)

    def profile(self) -> np.ndarray:
        """the profile the next push uses"""
        return self._profile.copy() if self._profile is not None else self.phi.copy()

    def frames_left(self) -> int:
        return self._learn if self._learn is not None else self.learn_left

    # ---- one step ----
    def push(self, chunk) -> np.ndarray:
        if self._reduction is not None:
            self.g = gain_floor(self._reduction)
        if self._profile is not None:
            self.phi = self._profile
        if self._learn is not None:
            self.learn_left = self.learn_total = self._learn
            self.learn_sum = np.zeros(NB)
        self._reduction = self._profile = self._learn = None
        start = len(self.x)
        self.x = np.concatenate([self.x, np.asarray(chunk, np.float32).astype(np.float64)])
        f1 = len(self.x) // H
        need = f1 * H + D
        if len(self.acc) < need:
            self.acc = np.concatenate([self.acc, np.zeros(need - len(self.acc))])
        phi, learned = self.phi, False
        zero = phi == 0.0
        safe = np.where(zero, 1.0, phi)
        for m in range(self.frames_done, f1):
            X = frame_spectrum(self.x, m)
            P = X.real * X.real + X.imag * X.imag
            xi = ALPHA * (self.G * self.G) * self.Pp / safe + (1.0 - ALPHA) * np.maximum(P / safe - 1.0, 0.0)
            G = np.where(zero, 1.0, np.fmax(xi / (1.0 + xi), self.g))
            y = WINDOW * np.fft.irfft(G * X, N)
            s = m * H - (N - H)
            self.acc[s + D:s + D + N] += y
            self.G, self.Pp = G, P
            if self.learn_left > 0:
                self.learn_sum = self.learn_sum + P
                self.learn_left -= 1
                learned = self.learn_left == 0
        self.frames_done = f1
        if learned:
            self.phi = self.learn_sum / self.learn_total
        # the samples t = start - D .. len(x) - D - 1 of z, zero before 0
        t = np.arange(start - D, len(self.x) - D)
        z = np.where(t < 0, 0.0, 0.5 * self.acc[t + D])
        return z.astype(np.float32)


def denoise(x, reduction_db: float, phi: Optional[np.ndarray] = None) -> np.ndarray:
    """The whole-signal filter (ryk_denoise): a fresh state, x zero outside [0, n), n samples out, no delay."""
    x = np.asarray(x, np.float32)
    o = DenoiseOracle(reduction_db, phi)
    return o.push(np.concatenate([x, np.zeros(D, np.float32)]))[D:]
