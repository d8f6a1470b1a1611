"""Stage-2 padded tail on the device: a forward that skips the encoder rows repeating the padded tail (mode 3 of
ryk_test_stage2_forward) runs on NaN-filled buffers.  Its kept rows must be finite and bitwise equal to the full forward's: a skipped
row that any computed pixel read would carry NaN into the output, and a remapped load box that read other values than the row it
stands for would change bits."""
import numpy as np
import pytest

from realtime_yukarin_b200 import engine as eng
from tests.session_geometry import stage2_cases
from tests.test_gpu_stage2_band import W, _load_stage2

# (Tp, Tw, kept ranges): the session shapes at 0.3 s (headline), 0.1 s and 1.0 s chunks, a window whose third encoder layer
# (split K) skips rows too, a kept band at the end of the window, a group of two members with different kept rows, and the session
# geometries of tests/session_geometry.py (Tp 128 to 1920)
CASES = ([(384, 260, [(100, 60)]), (256, 220, [(100, 20)]), (512, 400, [(100, 200)]), (640, 400, [(200, 200)]),
          (384, 300, [(240, 60)]), (384, 260, [(100, 60), (80, 100)])]
         + [(Tp, Tw, [(kb, kl)]) for Tp, kb, kl, Tw in stage2_cases()])


def _padded_input(B, Tp, Tw, seed):
    """rows >= Tw hold the per-column minimum of the window's rows, as the session's stage-2 prologue pads them"""
    rng = np.random.default_rng(seed)
    x = (-9.0 + 2.5 * rng.standard_normal((B, Tp, W))).astype(np.float32)
    x[:, Tw:] = x[:, :Tw].min(axis=1, keepdims=True)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize('Tp,Tw,keeps', CASES)
def test_tail_skip_forward_on_nan_buffers(engine, full_models, Tp, Tw, keeps):
    _load_stage2(engine, full_models)
    kb = min(k[0] for k in keeps)
    ke = max(k[0] + k[1] for k in keeps)
    # the case skips rows, unless one row of padding leaves no two rows equal (the forward must then be the full one)
    assert eng.stage2_tail_rows(Tp, W, Tw, kb, ke - kb)[:, 1].any() == (Tp - Tw > 1)
    x = _padded_input(len(keeps), Tp, Tw, Tp * 1000 + Tw)
    full = engine.test_stage2_forward(x, mode=0)
    assert np.isfinite(full).all()
    tail = engine.test_stage2_forward(x, keep=keeps, mode=3, tw=Tw)
    for j, (b, n) in enumerate(keeps):
        assert np.isfinite(tail[j, b:b + n]).all(), (j, b, n)
        assert np.array_equal(tail[j, b:b + n], full[j, b:b + n]), (j, b, n)
    assert np.isnan(tail[:, :kb]).all() and np.isnan(tail[:, ke:]).all()
