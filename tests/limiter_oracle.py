"""The FP64 numpy restatement of the output limiter (DESIGN.md DECIDE L1-L4), without a GPU.

    g0[u] = 1 if G |y[u]| <= c else c / (G |y[u]|)        (1 for u < 0),  c = 10^(ceiling_db / 20)
    m[s]  = min of g0[u] over u in [s - R, s + L - 1]
    g[t]  = (m[t - L + 1] + ... + m[t]) / L, summed in ascending s from 0.0
    z[t]  = g[t] y[t]

`limit` is the whole signal with y zero outside [0, n) and no delay; `LimiterStream` is a session's limiter step by step: each push of
n samples returns n samples of concat(zeros(L), z), and the settings of a push apply to g0 of the samples it brings."""
import numpy as np


def shape(rate, lookahead_ms, hold_ms):
    """(L, R) in samples at `rate`, rounded half to even as the library rounds them"""
    return max(1, round(lookahead_ms * rate / 1000)), round(hold_ms * rate / 1000)


def ceiling(ceiling_db):
    """c = 10^(ceiling_db / 20) through the C library's pow, as the library computes it (elementwise for an array)"""
    if np.ndim(ceiling_db):
        return np.array([ceiling(float(v)) for v in np.ravel(ceiling_db)]).reshape(np.shape(ceiling_db))
    return 10.0 ** (float(ceiling_db) / 20.0)


def gain0(y, c, gain):
    """g0 of the samples y: 1 where G |y| <= c, else c / (G |y|)"""
    a = gain * np.abs(np.asarray(y, np.float64))
    out = np.ones_like(a)
    np.divide(c, a, out=out, where=a > c)
    return out


def sliding_min(a, w):
    """min of a[q : q + w] for q = 0 .. len(a) - w, by blocked prefix / suffix minima (van Herk / Gil-Werman): the block of q ends where
    the block of q + w - 1 begins, so the window is the suffix of the one and the prefix of the other.  Minima are exact."""
    a = np.asarray(a, np.float64)
    n = len(a)
    blocks = -(-n // w)
    pad = np.full(blocks * w, np.inf)
    pad[:n] = a
    rows = pad.reshape(blocks, w)
    prefix = np.minimum.accumulate(rows, axis=1).ravel()
    suffix = np.minimum.accumulate(rows[:, ::-1], axis=1)[:, ::-1].ravel()
    q = np.arange(n - w + 1)
    return np.minimum(suffix[q], prefix[q + w - 1])


def box_mean(m, L, n):
    """g[j] = (m[j] + ... + m[j + L - 1]) / L for j < n, summed term by term in ascending order from 0.0"""
    acc = np.zeros(n)
    for k in range(L):
        acc = acc + m[k:k + n]
    return acc / L


def limit(y, rate, lookahead_ms=5.0, hold_ms=50.0, ceiling_db=-1.0, gain=1.0, return_gain=False):
    """z of the whole signal y (zero outside [0, n)), no delay; with return_gain also g.  ceiling_db and gain may also be arrays of
    n per-sample settings (those of g0[u])."""
    y = np.asarray(y, np.float64)
    n = len(y)
    L, R = shape(rate, lookahead_ms, hold_ms)
    u0 = -(R + 2 * L - 2)                       # g0 over u in [u0, n + L - 1): every window of s in [-L + 1, n - 1]
    u = np.arange(u0, n + L - 1)
    inside = (u >= 0) & (u < n)
    g0 = np.ones(len(u))
    g0[inside] = gain0(y, ceiling(ceiling_db), np.asarray(gain, np.float64))
    m = sliding_min(g0, R + L)                  # m[i] is m[s] for s = i + u0 + R
    m = m[L - 1:L - 1 + n + L - 1]              # s = -L + 1 .. n - 1
    g = box_mean(m, L, n)
    z = g * y
    return (z, g) if return_gain else z


def meter(g):
    """(largest reduction in dB, samples with g < 1) of the gains g (L4)"""
    g = np.asarray(g, np.float64)
    lo = float(g.min()) if len(g) else 1.0
    return (-20.0 * np.log10(lo) if lo < 1.0 else 0.0), int(np.count_nonzero(g < 1.0))


class LimiterStream:
    """A session's limiter: the histories of y (L samples) and g0 (R + 2L - 1) and the position carried from push to push."""

    def __init__(self, rate, lookahead_ms=5.0, hold_ms=50.0):
        self.L, self.R = shape(rate, lookahead_ms, hold_ms)
        self.hist_g0 = np.ones(self.R + 2 * self.L - 1)     # g0 = 1 before the stream
        self.hist_y = np.zeros(self.L)
        self.pos = 0
        self.set(-1.0, 1.0)
        self.last_meter = (0.0, 0)

    def set(self, ceiling_db, gain):
        """the settings of the next push"""
        self.c, self.gain = ceiling(ceiling_db), float(gain)

    def push(self, y):
        """n samples of y in, n samples of concat(zeros(L), z) out"""
        y = np.asarray(y, np.float64)
        n, L, R = len(y), self.L, self.R
        a = np.concatenate([self.hist_g0, gain0(y, self.c, self.gain)])
        yc = np.concatenate([self.hist_y, y])
        out = np.zeros(n)
        g = np.ones(n)
        if n:
            m = sliding_min(a, R + L)[:n + L - 1]
            g = box_mean(m, L, n)
            out = g * yc[:n]
            lead = self.pos + np.arange(n) - L < 0      # the leading zeros of the delay
            out[lead] = 0.0
            g[lead] = 1.0
        self.last_meter = meter(g)
        self.hist_g0 = a[n:]
        self.hist_y = yc[n:]
        self.pos += n
        return out
