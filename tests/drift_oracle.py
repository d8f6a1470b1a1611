"""The FP64 numpy restatement of the clock drift stage (DESIGN.md §4l, DECIDE D1-D3), without a GPU.

The stage reads z = concat(zeros(W), x) at positions q_m = inc_0 + ... + inc_(m-1) (q_0 = 0) in units of 2^-32 samples, with
inc = llrint(2^32 / (1 + ppm 1e-6)) of the setting in force.  For q = i 2^32 + f (0 <= f < 2^32):

    phi = f >> 23,  w = (f & (2^23 - 1)) 2^-23
    c_t = T[(2W - 1 - t) P + phi] + w (T[(2W - 1 - t) P + phi + 1] - T[(2W - 1 - t) P + phi])       t = 0 .. 2W - 1
    y_m = sum over t of c_t z[i - W + 1 + t], in ascending t from 0.0

with z zero before 0.  Output m is emitted once z[i + W] has arrived, so after N input samples the stage has emitted every m with
q_m < N 2^32.  Python ints hold the positions, so they never overflow here; `DriftStream` is the streaming object, `resample` the whole
signal followed by W zeros."""
import math

import numpy as np

from realtime_yukarin_b200.wave_io import DRIFT_HALF_WIDTH as W, DRIFT_PHASES as P, drift_filter

ONE = 1 << 32


def inc_of(ppm):
    """llrint(2^32 / (1 + ppm 1e-6)) with the same FP64 operations as the library (Python's round is half to even, like llrint)"""
    return int(round(4294967296.0 / (1.0 + float(ppm) * 1e-6)))


def capacity(n, max_ppm):
    """the documented bound of the outputs of one push of n samples"""
    return n + math.ceil(n * float(max_ppm) * 1e-6) + 2


def count(n, pos, inc):
    """outputs of a push of n samples from relative position pos: those with pos + k inc < n 2^32"""
    num = n * ONE - pos
    return max(0, -(-num // inc))


def outputs(b, pos, inc, k, table):
    """outputs 0 .. k - 1 of a push from relative position pos over b = the 2W kept samples followed by the push's samples"""
    return at_positions(b, np.int64(pos) + np.int64(inc) * np.arange(k, dtype=np.int64), table)


def at_positions(b, q, table):
    """the outputs at positions q (int64, 2^-32 samples) of z over b = concat(zeros(W), z), b[s] = z[s - W]"""
    q = np.asarray(q, np.int64)
    k = len(q)
    i = q >> 32
    f = q & (ONE - 1)
    phi = f >> 23
    w = (f & ((1 << 23) - 1)).astype(np.float64) * 2.0 ** -23
    acc = np.zeros(k)
    for t in range(2 * W):
        base = (2 * W - 1 - t) * P + phi
        c = table[base] + w * (table[base + 1] - table[base])
        acc = acc + c * b[i + 1 + t]
    return acc


class DriftStream:
    """A drift object: position relative to the samples consumed, totals, the last 2W samples and the setting."""

    def __init__(self, ppm=0.0, table=None):
        self.table = drift_filter() if table is None else np.asarray(table, np.float64)
        self.pos = 0
        self.consumed = 0
        self.produced = 0
        self.hist = np.zeros(2 * W)
        self.set(ppm)

    def set(self, ppm):
        """the setting of the next push"""
        self.ppm = float(ppm)
        self.inc = inc_of(ppm)

    def push(self, x):
        x = np.asarray(x, np.float64)
        n = len(x)
        b = np.concatenate([self.hist, x])
        k = count(n, self.pos, self.inc)
        y = outputs(b, self.pos, self.inc, k, self.table) if k else np.zeros(0)
        self.pos += k * self.inc - n * ONE
        self.hist = b[n:]
        self.consumed += n
        self.produced += k
        return y


def resample(x, ppm, table=None):
    """the whole signal from a fresh state, followed by W zeros"""
    s = DriftStream(ppm, table)
    return s.push(np.concatenate([np.asarray(x, np.float64), np.zeros(W)]))


def positions(incs):
    """absolute positions q_m of outputs whose increments are incs (q_0 = 0)"""
    return np.concatenate([[0], np.cumsum(np.asarray(incs, dtype=object))])[:len(incs)]
