"""Stage-2 padded tail: a session pads its Tw-frame window to Tp rows with one repeated row, so every encoder layer has a run of
equal output rows that depend on nothing but that padding.  The encoder computes the first rows of each run and skips the rest
(unet_derive_tail in csrc/unet.cu); the next layer reads a load box that lies wholly inside the run from the run's first rows.

The library's table is checked against an independent walk: runs found by following which input rows every output row reads,
and the skip as the longest range of whole tile rows that no load box crossing the run's end, no representative row and no
decoder read touches.
"""
import numpy as np
import pytest

from realtime_yukarin_b200 import engine as eng
from tests.session_geometry import stage2_cases
from tests.test_gpu_stage2_band import CASES, W, _python_bands, _tile_rows

CIN1_ROWS = 8          # output rows per CTA of the first layer's kernel (k_conv3x3_cin1)


def _runs(Tp, Tw):
    """[(lo, hi)] per encoder layer 0..7: the rows equal to each other because they read only padding (lo > hi: none)"""
    ident = [('x', r) for r in range(Tw)] + [('x', 'pad')] * (Tp - Tw)
    runs = []
    for i in range(8):
        k, s, p = (3, 1, 1) if i == 0 else (4, 2, 1)
        Hout = Tp >> i
        ident = [tuple(ident[o * s - p + t] if 0 <= o * s - p + t < len(ident) else None for t in range(k)) for o in range(Hout)]
        groups = {}
        for r, v in enumerate(ident):
            groups.setdefault(v, []).append(r)
        rep = [g for g in groups.values() if len(g) > 1]
        assert len(rep) <= 1
        if rep:
            g = rep[0]
            assert g == list(range(g[0], g[-1] + 1))
            runs.append((g[0], g[-1]))
        else:
            runs.append((1, 0))
    return runs


def _python_tail(Tp, Tw, keep_begin, keep_len):
    bands = _python_bands(Tp, keep_begin, keep_len)
    runs = _runs(Tp, Tw)
    out = np.zeros((16, 4), np.int32)
    for i in range(6, -1, -1):
        lo, hi = runs[i]
        if lo > hi:
            continue
        Hout = Tp >> i
        th = CIN1_ROWS if i == 0 else _tile_rows(W >> i)
        nth = _tile_rows(W >> (i + 1))
        span = 2 * (nth - 1) + 1
        bad = np.ones(Hout, bool)
        bad[lo:hi + 1] = False
        bad[lo:lo + span] = True                               # representative rows
        n_skip = out[i + 1, :2]
        for t in range(-(-(Tp >> (i + 1)) // nth)):
            if n_skip[0] <= t * nth < n_skip[1]:
                continue
            for ty in range(4):
                s = 2 * t * nth + ty - 1
                if not (lo <= s and s + span - 1 <= hi):
                    bad[max(s, 0):max(s + span, 0)] = True
        y0, y1 = bands[15 - i]                                  # decoder layer reading this output: rows m - 1 .. m + 1
        bad[max(y0 - 1, 0):y1 + 1] = True
        best = (0, 0)
        for a in range(0, Hout, th):
            b = a
            while b + th <= Hout and not bad[b:b + th].any():
                b += th
            if b - a > best[1] - best[0]:
                best = (a, b)
        if best[1] > best[0]:
            out[i, :2] = best
            out[i + 1, 2:] = (lo, hi + 1)
    return out


def _tws(Tp, kb, kl):
    """windows padded to Tp: a whole block, half a block and one row of padding, and the session geometries' own"""
    return sorted({max(Tp - 128, 1), Tp - 64, Tp - 1} | {c[3] for c in stage2_cases() if c[:3] == (Tp, kb, kl)})


@pytest.mark.parametrize('Tp,kb,kl', CASES)
def test_tail_table_matches_independent_walk(Tp, kb, kl):
    for Tw in _tws(Tp, kb, kl):
        got = eng.stage2_tail_rows(Tp, W, Tw, kb, kl)
        want = _python_tail(Tp, Tw, kb, kl)
        assert np.array_equal(got, want), (Tw, got.tolist(), want.tolist())


def test_tail_table_headline_shape():
    """0.3 s chunks with 0.5 s extras: 260 frames padded to 384 rows, rows [100, 160) kept"""
    t = eng.stage2_tail_rows(384, W, 260, 100, 60)
    assert t[:4].tolist() == [[264, 376, 0, 0], [132, 191, 261, 383], [69, 93, 131, 191], [0, 0, 66, 95]]
    assert not t[4:].any()


def test_tail_skip_shrinks_away_from_decoder_reads():
    """a kept band at the end of the window: the decoder reads encoder rows inside the runs, which stay computed"""
    for Tp, Tw, kb, kl in [(384, 300, 240, 60), (256, 250, 200, 50), (128, 127, 90, 37)]:
        t = eng.stage2_tail_rows(Tp, W, Tw, kb, kl)
        bands = eng.stage2_row_bands(Tp, W, kb, kl)
        for i in range(7):
            y0, y1 = bands[15 - i]
            r0, r1 = max(y0 - 1, 0), y1 + 1
            assert t[i, 1] <= r0 or t[i, 0] >= r1, (Tp, Tw, kb, kl, i, t[i].tolist(), (r0, r1))
