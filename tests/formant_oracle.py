"""FP64 reference of the formant warp (DESIGN.md DECIDE F1) for the tests, on top of the oracle, which it leaves as it is: the warp
acts on stage 2's log-spectrum between the edge pad and exp, where the device's stage-2 epilogue applies it."""
import functools
from unittest import mock

import numpy as np

from oracle import nets as onets
from oracle import pipeline as opipe


def formant_warp(y: np.ndarray, ratio: float) -> np.ndarray:
    """(T, nb - 1) network log rows -> (T, nb) float32: the edge-padded rows L[j] = y[min(j, nb - 2)] read at x = k / ratio, linearly
    interpolated in FP64 and held at L[nb - 1] from x >= nb - 1 on.  Ratio 1 is the edge pad itself."""
    L = np.pad(np.asarray(y, np.float32), [(0, 0), (0, 1)], mode='edge')
    if ratio == 1.0:
        return L
    nb = L.shape[1]
    x = np.arange(nb, dtype=np.float64) / float(ratio)
    top = x >= nb - 1
    i = np.where(top, 0, np.floor(x)).astype(np.int64)
    w = x - i
    Ld = L.astype(np.float64)
    out = (1.0 - w) * Ld[:, i] + w * Ld[:, np.minimum(i + 1, nb - 1)]
    out[:, top] = Ld[:, nb - 1:nb]
    return out.astype(np.float32)


def stage2_convert(sp: np.ndarray, p, backend: str = 'numpy', formant_ratio: float = 1.0) -> np.ndarray:
    """oracle.nets.stage2_convert with the warp between the edge pad and exp; ratio 1 is that function."""
    if formant_ratio == 1.0:
        return onets.stage2_convert(sp, p, backend)
    x = np.asarray(sp, dtype=np.float32)
    pad = 128 - len(x) % 128
    x = np.pad(x, [(0, pad), (0, 0)], mode='minimum')
    x = np.log(x)[:, :-1][np.newaxis]
    y = onets.unet_forward(x, p, 2, backend)[0]
    return np.exp(formant_warp(y, formant_ratio))[:-pad].astype(np.float32)


class FormantStreamOracle(opipe.StreamOracle):
    """StreamOracle whose stage 2 warps the envelope by `formant_ratio`, which a test may change between pushes."""
    formant_ratio = 1.0

    def push(self, chunk):
        if self.formant_ratio == 1.0:
            return super().push(chunk)
        with mock.patch.object(opipe.nets, 'stage2_convert', functools.partial(stage2_convert, formant_ratio=self.formant_ratio)):
            return super().push(chunk)
