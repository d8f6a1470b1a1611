"""FP64 numpy reference of the echo canceller (DESIGN.md DECIDE E1-E4) for the tests.

EchoOracle is the streaming canceller a session runs: push(mic, far) takes the model-rate microphone chunk of a step and the far-end
samples played while it was recorded, and returns the filtered chunk of concat(zeros(D), z).  It frames both signals as the noise
suppression does (tests/denoise_oracle.py), cancels per bin with a two-path NLMS filter over the frames of the far end, applies the
residual suppression and, with a noise profile, the noise suppression's gain scan on the result, and overlap-adds the frames in
ascending order.  echo_cancel() is the whole-signal call (ryk_echo_cancel).  A chunked stream equals the whole signal exactly.

`two_path=False` is the single NLMS filter (the background filter produces the output and no copy is made): the tests show that the
two-path control keeps more of the near-end voice during double talk."""
from typing import Optional

import numpy as np

from .denoise_oracle import ALPHA, D, H, N, NB, WINDOW, frame_spectrum, gain_floor

MU = 0.5                 # NLMS step (E2)
DELTA = 1e-6             # NLMS regularisation (E2)
LAMBDA = 0.9             # power smoothing (E3, E4)
COPY_RATIO = 0.5         # B -> F when S_b < COPY_RATIO S_f and S_b < S_d ...
COPY_FRAMES = 3          # ... for this many consecutive frames (E3)
RESET_RATIO = 4.0        # F -> B, no update, when S_b > RESET_RATIO S_f (E3)
DIVERGED_RATIO = 1.0     # F -> 0 when S_f > DIVERGED_RATIO S_d: the output would be louder than the microphone (E3)
RHO = 1.0                # residual suppression: G = max(g_e, 1 - RHO Yhat / (Ehat + EPS)) (E4)
EPS = 1e-12
MAX_TAPS, MAX_DELAY = 64, 256


class EchoOracle:
    """The session's canceller, step by step.  Frame m is processed in the push whose samples hold its last sample m H + H - 1."""

    def __init__(self, taps: int = 32, delay_frames: int = 0, suppression_db: float = 0.0, reduction_db: float = 20.0,
                 phi: Optional[np.ndarray] = None, two_path: bool = True):
        assert 1 <= taps <= MAX_TAPS and 0 <= delay_frames <= MAX_DELAY
        self.P, self.d, self.two_path = int(taps), int(delay_frames), two_path
        self.ge = gain_floor(suppression_db)
        self.g_dn = gain_floor(reduction_db)
        self.phi = None if phi is None else np.array(phi, np.float64)
        self.B = np.zeros((NB, self.P), complex)
        self.F = np.zeros((NB, self.P), complex)
        self.Xt = np.zeros((NB, self.P), complex)          # X_{m-d-p} of the next frame's taps, p = 0 .. P - 1
        self.far_frames = []                               # X_m of every far-end frame so far
        self.Sb, self.Sf, self.Sd, self.Yh, self.Eh = (np.zeros(NB) for _ in range(5))
        self.cnt = np.zeros(NB, np.int64)
        self.G_dn, self.P_dn = np.ones(NB), np.zeros(NB)
        self.mic, self.far = np.zeros(0), np.zeros(0)
        self.acc = np.zeros(D)
        self.frames_done = 0
        self.copies = np.zeros(NB, np.int64)               # B -> F copies per bin (the GPU test reports bins whose count differs)
        self.stats = (0, 0.0, 0.0)                          # frames, sum |D|^2, sum |Z|^2 of the last push
        self._suppression = None

    def set_suppression(self, db: float):
        """from the next push on"""
        self._suppression = float(db)

    def erle_db(self) -> float:
        _, sd, sz = self.stats
        return 10.0 * np.log10(sd / sz)

    def push(self, mic, far) -> np.ndarray:
        if self._suppression is not None:
            self.ge = gain_floor(self._suppression)
            self._suppression = None
        mic, far = np.asarray(mic, np.float32), np.asarray(far, np.float32)
        assert len(mic) == len(far)
        start = len(self.mic)
        self.mic = np.concatenate([self.mic, mic.astype(np.float64)])
        self.far = np.concatenate([self.far, far.astype(np.float64)])
        f1 = len(self.mic) // H
        need = f1 * H + D
        if len(self.acc) < need:
            self.acc = np.concatenate([self.acc, np.zeros(need - len(self.acc))])
        lam = LAMBDA
        sum_d = sum_z = 0.0
        for m in range(self.frames_done, f1):
            Dm = frame_spectrum(self.mic, m)
            self.far_frames.append(frame_spectrum(self.far, m))
            q = m - self.d
            self.Xt[:, 1:] = self.Xt[:, :-1]
            self.Xt[:, 0] = self.far_frames[q] if q >= 0 else 0.0
            Xt = self.Xt
            Px = np.sum(Xt.real * Xt.real + Xt.imag * Xt.imag, axis=1)
            Yb = np.sum(self.B * Xt, axis=1)
            Yf = np.sum(self.F * Xt, axis=1) if self.two_path else Yb
            Eb, Ef = Dm - Yb, Dm - Yf
            self.Sb = lam * self.Sb + (1 - lam) * np.abs(Eb) ** 2
            self.Sf = lam * self.Sf + (1 - lam) * np.abs(Ef) ** 2
            self.Sd = lam * self.Sd + (1 - lam) * np.abs(Dm) ** 2
            self.Yh = lam * self.Yh + (1 - lam) * np.abs(Yf) ** 2
            self.Eh = lam * self.Eh + (1 - lam) * np.abs(Ef) ** 2
            G = np.fmax(self.ge, 1.0 - RHO * self.Yh / (self.Eh + EPS))
            Z = G * Ef
            sum_d += float(np.sum(np.abs(Dm) ** 2))
            sum_z += float(np.sum(np.abs(Z) ** 2))
            # the filters, in this order: clear a diverged F, reset B from F (no update), else count, copy B into F, update B
            upd = self.B + (MU / (Px + DELTA))[:, None] * Eb[:, None] * np.conj(Xt)
            if self.two_path:
                self.F = np.where((self.Sf > DIVERGED_RATIO * self.Sd)[:, None], 0.0, self.F)
                reset = self.Sb > RESET_RATIO * self.Sf
                self.cnt = np.where(reset, 0, np.where((self.Sb < COPY_RATIO * self.Sf) & (self.Sb < self.Sd), self.cnt + 1, 0))
                copy = self.cnt >= COPY_FRAMES
                self.copies += copy
                self.F = np.where(copy[:, None], self.B, self.F)
                self.cnt = np.where(copy, 0, self.cnt)
                self.B = np.where(reset[:, None], self.F, upd)
            else:
                self.B = upd
            if self.phi is not None:                       # the noise suppression's gain scan (N2) on Z
                Pz = Z.real * Z.real + Z.imag * Z.imag
                zero = self.phi == 0.0
                safe = np.where(zero, 1.0, self.phi)
                xi = ALPHA * (self.G_dn * self.G_dn) * self.P_dn / safe + (1.0 - ALPHA) * np.maximum(Pz / safe - 1.0, 0.0)
                self.G_dn = np.where(zero, 1.0, np.fmax(xi / (1.0 + xi), self.g_dn))
                self.P_dn = Pz
                Z = self.G_dn * Z
            y = WINDOW * np.fft.irfft(Z, N)
            s = m * H - (N - H)
            self.acc[s + D:s + D + N] += y
        self.stats = (f1 - self.frames_done, sum_d, sum_z)
        self.frames_done = f1
        t = np.arange(start - D, len(self.mic) - D)
        z = np.where(t < 0, 0.0, 0.5 * self.acc[t + D])
        return z.astype(np.float32)


def echo_cancel(mic, far, taps: int = 32, delay_frames: int = 0, suppression_db: float = 0.0, reduction_db: float = 20.0,
                phi: Optional[np.ndarray] = None, two_path: bool = True, oracle: bool = False):
    """The whole-signal call (ryk_echo_cancel): a fresh state, both signals zero outside [0, n), n samples out, no delay.  With
    oracle=True also returns the EchoOracle that ran it."""
    mic, far = np.asarray(mic, np.float32), np.asarray(far, np.float32)
    o = EchoOracle(taps, delay_frames, suppression_db, reduction_db, phi, two_path)
    z = o.push(np.concatenate([mic, np.zeros(D, np.float32)]), np.concatenate([far, np.zeros(D, np.float32)]))[D:]
    return (z, o) if oracle else z


# ---- synthetic rooms for the tests ----
def room_ir(delay_ms: float, fs: int = 24000, tail_ms: float = 100.0, gain: float = 0.5, seed: int = 0) -> np.ndarray:
    """a bulk delay, then a seeded exponentially decaying noise tail of time constant tail_ms / 3, scaled to an L2 norm of gain"""
    d = int(round(delay_ms * fs / 1000))
    n = int(round(tail_ms * fs / 1000))
    tail = np.random.default_rng(seed).standard_normal(n) * np.exp(-3.0 * np.arange(n) / n)
    return np.concatenate([np.zeros(d), gain * tail / np.linalg.norm(tail)])


def echo_of(far, ir) -> np.ndarray:
    """what the microphone picks up of `far` through the room `ir`, as long as far (float64)"""
    return np.convolve(np.asarray(far, np.float64), ir)[:len(far)]


def level_db(x, ref) -> float:
    """10 log10 of the power of x over the power of ref"""
    x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
    return 10.0 * np.log10(np.mean(x * x) / np.mean(ref * ref))
