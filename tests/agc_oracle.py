"""FP64 numpy restatement of the automatic gain control (DESIGN.md §4j, DECIDE A1-A4): the whole-signal `agc` and the streaming
`AgcStream`, written independently of each other so that each checks the other.

Every operation is + - * /, sqrt, min or max in FP64, so the device's explicit round-to-nearest arithmetic gives these bits.  Block
sums are sequential (np.cumsum, not np.sum, which adds pairwise).  The host values use Python's math, which calls the same libm as
the library's host code.
"""
import math

import numpy as np

B = 256                                   # model samples per level block (A1)
NAMES = ('target', 'gate', 'gmax', 'ginv', 'a', 's_up', 's_dn')


def params(fs, target_db=-26.0, max_gain_db=20.0, gate_db=-50.0):
    """the linear values the device uses (A2), in the order of ryk_session_get_agc's `linear`"""
    gmax = math.pow(10.0, max_gain_db / 20.0)
    return dict(target=math.pow(10.0, target_db / 10.0), gate=math.pow(10.0, gate_db / 10.0), gmax=gmax, ginv=1.0 / gmax,
                a=-math.expm1(-B / (0.4 * fs)), s_up=math.pow(10.0, 6.0 * B / (20.0 * fs)), s_dn=math.pow(10.0, -24.0 * B / (20.0 * fs)))


def _block_power(sq):
    return float(np.cumsum(sq)[-1]) / B


def _gain_step(P, p, E, started, g):
    """one block of the A2 recursion: (E, started, g, active)"""
    if not p > P['gate']:
        return E, started, g, False
    E = E + P['a'] * (p - E) if started else p
    want = min(max(math.sqrt(P['target'] / E), P['ginv']), P['gmax'])
    return E, True, min(max(want, g * P['s_dn']), g * P['s_up']), True


def _apply(x, pos, gains):
    """A3 over x, whose first sample sits at position pos of the block gains[0], gains[1] were not computed for: a sample in the k-th
    block from there ramps from gains[k] to gains[k + 1] (from the start: gains[m] = g_{m-2})"""
    s = pos + np.arange(len(x))
    m = s // B
    j = s - m * B
    ga, gb = gains[m], gains[m + 1]
    g = ga + (gb - ga) * ((j + 1) / B)
    return (g * x.astype(np.float64)).astype(np.float32)


def agc(x, fs, target_db=-26.0, max_gain_db=20.0, gate_db=-50.0, return_gain=False):
    """The whole signal from a fresh state.  A setting may be an array with one value per completed block (block m uses entry m).
    With return_gain also the gains g_m of the completed blocks and their active flags."""
    x = np.asarray(x, np.float32)
    nb = len(x) // B
    settings = [np.broadcast_to(np.asarray(v, np.float64), (nb,)) for v in (target_db, max_gain_db, gate_db)]
    xd = x.astype(np.float64)
    E, started, g = 0.0, False, 1.0
    gains, active = np.ones(nb + 2), np.zeros(nb, bool)
    for m in range(nb):
        P = params(fs, *(float(v[m]) for v in settings))
        seg = xd[m * B:(m + 1) * B]
        E, started, g, active[m] = _gain_step(P, _block_power(seg * seg), E, started, g)
        gains[m + 2] = g
    z = _apply(x, 0, gains)
    return (z, gains[2:], active) if return_gain else z


class AgcStream:
    """A session's gain control step by step: set() changes the settings of the next push; push(x) returns z for x at once."""

    def __init__(self, fs, target_db=-26.0, max_gain_db=20.0, gate_db=-50.0):
        self.fs = fs
        self.set(target_db, max_gain_db, gate_db)
        self.pos, self.E, self.started, self.g1, self.g2 = 0, 0.0, False, 1.0, 1.0
        self.hist = np.zeros(0, np.float32)
        self.last_meter = (-math.inf, 0.0, 0)

    def set(self, target_db, max_gain_db, gate_db):
        self.P = params(self.fs, target_db, max_gain_db, gate_db)

    def push(self, x):
        x = np.asarray(x, np.float32)
        buf = np.concatenate([self.hist, x]).astype(np.float64)
        nc = len(buf) // B
        if nc:
            powers = (buf[:nc * B] * buf[:nc * B]).reshape(nc, B).cumsum(axis=1)[:, -1] / B
        gains = [self.g2, self.g1]
        E, started, g, n_active = self.E, self.started, self.g1, 0
        for i in range(nc):
            E, started, g, act = _gain_step(self.P, float(powers[i]), E, started, g)
            n_active += act
            gains.append(g)
        # gains[i] = g_{m0 - 2 + i}: a sample of block m uses gains[m - m0] and gains[m - m0 + 1]
        z = _apply(x, self.pos % B, np.array(gains))
        self.pos += len(x)
        self.E, self.started, self.g1, self.g2 = E, started, gains[-1], gains[-2]
        self.hist = np.asarray(buf[nc * B:], np.float32)
        self.last_meter = meter(E, started, g, n_active)
        return z


def meter(E, started, g, active):
    """(10 log10 E or -inf before any active block, 20 log10 g, active blocks of the step), the logs taken as the host takes them"""
    return (10.0 * math.log10(E) if started else -math.inf, 20.0 * math.log10(g), int(active))


def level_db(x):
    """mean square of x in dB of full scale"""
    x = np.asarray(x, np.float64)
    return 10.0 * math.log10(float(np.mean(x * x)))
