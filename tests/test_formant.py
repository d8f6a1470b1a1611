"""Host side of the formant ratio, without a GPU: the FP64 reference warp against numpy.interp, where it moves an envelope, the
semitone arithmetic and argument rules of Engine.session_set_formant, the staged VoiceChanger's control and run.py --formant."""
import math
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import nets as onets
from realtime_yukarin_b200 import engine as eng
from realtime_yukarin_b200 import run

from .formant_oracle import formant_warp, stage2_convert

NB = 513


def _rows(seed=0, T=4):
    return np.random.default_rng(seed).normal(-6.0, 2.0, size=(T, NB - 1)).astype(np.float32)


@pytest.mark.parametrize('r', [0.5, 0.8, 2 ** (-3 / 12), 1.0, 2 ** (5 / 12), 1.25, 2.0])
def test_warp_is_numpy_interp(r):
    y = _rows()
    L = np.pad(y, [(0, 0), (0, 1)], mode='edge')
    want = np.stack([np.interp(np.arange(NB) / r, np.arange(NB), row.astype(np.float64)) for row in L]).astype(np.float32)
    got = formant_warp(y, r)
    assert got.dtype == np.float32 and got.shape == (len(y), NB)
    np.testing.assert_array_max_ulp(got, want, maxulp=1)
    np.testing.assert_allclose(np.exp(got), np.exp(want), rtol=1e-6)


def test_ratio_one_is_the_edge_pad_bitwise(small_models):
    y = _rows(1)
    assert np.array_equal(formant_warp(y, 1.0), np.pad(y, [(0, 0), (0, 1)], mode='edge'))
    p2 = onets.load_npz(small_models['stage2_model_path'])
    sp = np.exp(np.random.default_rng(2).normal(-8.0, 1.0, size=(10, NB))).astype(np.float32)
    assert np.array_equal(stage2_convert(sp, p2, 'torch', formant_ratio=1.0), onets.stage2_convert(sp, p2, 'torch'))


def test_the_warp_is_applied_before_exp(small_models):
    """stage2_convert with a ratio is the oracle's output, warped in the log domain"""
    p2 = onets.load_npz(small_models['stage2_model_path'])
    sp = np.exp(np.random.default_rng(3).normal(-8.0, 1.0, size=(12, NB))).astype(np.float32)
    plain = onets.stage2_convert(sp, p2, 'torch')
    warped = stage2_convert(sp, p2, 'torch', formant_ratio=1.25)
    want = np.exp(formant_warp(np.log(plain.astype(np.float64))[:, :-1], 1.25))
    np.testing.assert_allclose(warped, want, rtol=1e-5)


def _bump(center=100.0, width=6.0):
    k = np.arange(NB - 1)
    return (-8.0 + 4.0 * np.exp(-0.5 * ((k - center) / width) ** 2)).astype(np.float32)[None]


@pytest.mark.parametrize('r', [0.8, 1.25])
def test_a_bump_moves_to_r_times_its_bin(r):
    got = formant_warp(_bump(), r)[0]
    assert abs(int(np.argmax(got)) - round(100 * r)) <= 1


def test_a_constant_row_stays_constant():
    y = np.full((2, NB - 1), -3.25, np.float32)
    for r in (0.5, 0.8, 1.25, 2.0):
        assert np.array_equal(formant_warp(y, r), np.full((2, NB), -3.25, np.float32))


@pytest.mark.parametrize('r', [0.5, 0.8, 2 ** (-3 / 12)])
def test_the_top_is_held_flat_below_one(r):
    y = _rows(4)
    got = formant_warp(y, r)
    top = np.arange(NB) >= (NB - 1) * r
    assert top.any()
    assert np.array_equal(got[:, top], np.repeat(y[:, -1:], top.sum(), axis=1))


def test_semitones_and_ratio():
    assert eng.formant_ratio(ratio=1.5) == 1.5
    assert eng.formant_ratio(semitones=12) == 2.0 and eng.formant_ratio(semitones=-12) == 0.5
    assert eng.formant_ratio(semitones=0) == 1.0
    assert eng.formant_ratio(semitones=4) == pytest.approx(2 ** (1 / 3), rel=1e-15)
    assert math.log2(eng.formant_ratio(semitones=-5)) * 12 == pytest.approx(-5, rel=1e-14)
    assert eng.FORMANT_RANGE == (eng.formant_ratio(semitones=-12), eng.formant_ratio(semitones=12))


class _Lib:
    """records the calls Engine.session_set_formant makes"""

    def __init__(self):
        self.calls = []

    def ryk_session_set_formant(self, h, sid, ratio):
        self.calls.append((sid, ratio.value))
        return 0


def test_session_set_formant_takes_exactly_one_of_ratio_and_semitones():
    fake = SimpleNamespace(lib=_Lib(), _h=None, _check=lambda rc: rc)
    set_formant = eng.Engine.session_set_formant
    set_formant(fake, 3, ratio=1.25)
    set_formant(fake, 4, semitones=-12)
    set_formant(fake, 5, 0.8)
    assert fake.lib.calls == [(3, 1.25), (4, 0.5), (5, 0.8)]
    for kw in (dict(), dict(ratio=1.2, semitones=3), dict(ratio=None, semitones=None)):
        with pytest.raises(ValueError):
            set_formant(fake, 3, **kw)
    assert len(fake.lib.calls) == 3


def test_the_fused_route_refuses_a_ratio():
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    sr = SimpleNamespace(config=SimpleNamespace(dataset=SimpleNamespace(param=SimpleNamespace(voice_param=SimpleNamespace(sample_rate=24000)))))
    assert VoiceChanger(None, sr, fused=True).formant_ratio == 1.0
    assert VoiceChanger(None, sr, formant_ratio=1.3).formant_ratio == 1.3
    with pytest.raises(ValueError):
        VoiceChanger(None, sr, fused=True, formant_ratio=1.3)


def test_the_staged_route_passes_the_ratio_to_stage_2():
    from realtime_yukarin_b200.models import SuperResolution
    seen = []

    class Eng:
        def stage2_convert(self, sp, **kw):
            seen.append(kw)
            return sp
    sr = SuperResolution.__new__(SuperResolution)
    sr.engine = Eng()
    x = np.ones((2, NB), np.float32)
    sr.convert(x)
    sr.convert(x, formant_ratio=0.9)
    assert seen == [{}, {'formant_ratio': 0.9}]


def test_run_flags():
    p = run.make_parser()
    a = p.parse_args([])
    assert a.formant == 0.0 and a.pitch == 0.0
    a = p.parse_args(['--wav_in', 'a.wav', '--formant', '3', '--pitch', '4'])
    assert a.formant == 3.0 and a.pitch == 4.0
    assert p.parse_args(['--formant', '-2.5']).formant == -2.5
    with pytest.raises(SystemExit):
        p.parse_args(['--formant', 'up'])
    assert '--formant' in p.format_help()
