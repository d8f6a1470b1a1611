"""The FP64 oracle of the pitch correction (tests/pitch_oracle.py, DESIGN.md §4m, DECIDE P1-P3) on synthetic contours, and the host
side of its settings: no device needed."""
import math

import numpy as np
import pytest

from realtime_yukarin_b200.engine import PITCH_SCALES, pitch_key, pitch_scale

from . import pitch_oracle as P

HOP = 5.0                    # ms per frame


def _contour(semis, a4=440.0):
    """f0 of a contour given in MIDI semitones (NaN: unvoiced -> 0)"""
    semis = np.asarray(semis, np.float64)
    return np.where(np.isnan(semis), 0.0, a4 * 2.0 ** ((semis - 69.0) / 12.0))


def _frames(seconds):
    return np.arange(round(seconds * 1000 / HOP))


def _vibrato(seconds=2.0, centre=64.0, depth=0.6, rate=5.5):
    t = _frames(seconds) * HOP / 1000
    return centre + depth * np.sin(2 * np.pi * rate * t)


def _glide(seconds=2.0, a=60.0, b=67.0):
    return np.linspace(a, b, len(_frames(seconds)))


def _gappy(seed=3):
    rng = np.random.default_rng(seed)
    s = 62.0 + np.cumsum(rng.normal(0, 0.08, 1200))
    for a in rng.integers(0, 1150, 14):
        s[a:a + rng.integers(3, 40)] = np.nan
    return s


CONTOURS = {'vibrato': _vibrato(), 'glide': _glide(), 'between': np.full(300, 64.5) + 0.04 * np.sin(np.arange(300) / 3.0),
            'gappy': _gappy(), 'silence': np.full(400, np.nan)}


@pytest.mark.parametrize('name', sorted(CONTOURS))
@pytest.mark.parametrize('settings', [dict(key=0, scale=PITCH_SCALES['major'], retune_ms=50.0, amount=1.0),
                                      dict(key=9, scale=PITCH_SCALES['minor'], retune_ms=0.0, amount=0.7, a4=432.0),
                                      dict(key=3, scale=0b000010000001, retune_ms=400.0, amount=1.0)])
def test_chunked_pushes_are_the_whole_signal(name, settings):
    f0 = _contour(CONTOURS[name])
    whole = P.pitch_correct(f0, HOP, **settings)
    rng = np.random.default_rng(len(name))
    for _ in range(3):
        st = P.PitchStream(HOP, **settings)
        cuts = np.sort(rng.integers(0, len(f0), 9))
        got = np.concatenate([st.push(part) for part in np.split(f0, cuts)])
        assert np.array_equal(got, whole), name
    assert np.array_equal(whole == 0, f0 == 0)


def test_amount_zero_is_the_identity_bit_for_bit():
    rng = np.random.default_rng(1)
    for name, semis in CONTOURS.items():
        f0 = _contour(semis)
        for retune in (0.0, 20.0, 1000.0):
            assert np.array_equal(P.pitch_correct(f0, HOP, 4, PITCH_SCALES['major'], 440.0, retune, 0.0).view(np.int64),
                                  f0.view(np.int64)), name
    odd = np.array([0.0, -0.0, -5.0, np.inf, np.nan, 1e-300, 5e-324, 1e300, 440.0])
    rng.shuffle(odd)
    assert np.array_equal(P.pitch_correct(odd, HOP, amount=0.0).view(np.int64), odd.view(np.int64))


def test_a_hard_chromatic_snap_puts_every_voiced_frame_on_a_note():
    for a4 in (440.0, 400.0, 480.0):
        f0 = _contour(_gappy(seed=int(a4)), a4=446.0)
        notes = []
        out = P.pitch_correct(f0, HOP, 0, 0xfff, a4, 0.0, 1.0, notes=notes)
        for i, n, s in notes:
            assert abs(out[i] / P.note_hz(n, a4) - 1.0) <= 1e-12, (a4, i, n, s)
        assert len(notes) == int(np.count_nonzero(f0))


def test_a_sustained_note_with_vibrato_keeps_its_note():
    # +-60 cents around E4 in C major: without hysteresis the crests (64.6) would go to F (65)
    semis = _vibrato(depth=0.6)
    notes = []
    out = P.pitch_correct(_contour(semis), HOP, 0, PITCH_SCALES['major'], 440.0, 0.0, 1.0, notes=notes)
    assert {n for _, n, _ in notes} == {64}
    assert max(P.nearest(s, 0, PITCH_SCALES['major']) for s in semis) == 65
    assert np.allclose(out, P.note_hz(64), rtol=1e-12, atol=0)
    # a slow retune leaves part of the vibrato: less than the input's, more than none
    soft = P.pitch_correct(_contour(semis), HOP, 0, PITCH_SCALES['major'], 440.0, 80.0, 1.0)
    dev = np.abs(12 * np.log2(soft / P.note_hz(64)))
    assert 0.05 < dev.max() < 0.6


def test_a_slow_glide_steps_through_each_note_once():
    semis = _glide(a=60.0, b=67.0)
    notes = []
    P.pitch_correct(_contour(semis), HOP, 0, 0xfff, 440.0, 0.0, 1.0, notes=notes)
    targets = np.array([n for _, n, _ in notes])
    assert targets[0] == 60 and targets[-1] == 67
    changes = np.flatnonzero(np.diff(targets))
    assert len(changes) == 7 and np.all(np.diff(targets)[changes] == 1)
    for j in changes:                      # the target moves up once s passes the old note by the hysteresis
        s_new = notes[j + 1][2]
        assert s_new - targets[j] >= P.HOLD and notes[j][2] - targets[j] < P.HOLD


def test_a_pitch_between_two_scale_notes_does_not_flap():
    semis = CONTOURS['between']
    notes = []
    P.pitch_correct(_contour(semis), HOP, 0, 0xfff, 440.0, 30.0, 1.0, notes=notes)
    assert len({n for _, n, _ in notes}) == 1
    nearest = [P.nearest(s, 0, 0xfff) for s in semis]
    assert len(set(nearest)) == 2, 'the contour crosses the midpoint'
    # an exact tie goes to the lower note
    assert P.nearest(64.5, 0, 0xfff) == 64
    assert P.nearest(66.0, 0, 0b000000000001) == 60      # C only: 66 is 6 from 60 and from 72


def test_no_glide_across_an_unvoiced_gap():
    semis = np.concatenate([np.full(100, 60.3), np.full(20, np.nan), np.full(100, 62.8)])
    notes = []
    out = P.pitch_correct(_contour(semis), HOP, 0, 0xfff, 440.0, 200.0, 1.0, notes=notes)
    assert np.all(out[100:120] == 0)
    first = 120
    assert abs(out[first] / P.note_hz(63) - 1) <= 1e-12     # c = d: straight on the note
    joined = P.pitch_correct(_contour(np.concatenate([semis[:100], semis[120:]])), HOP, 0, 0xfff, 440.0, 200.0, 1.0)
    assert abs(joined[100] / P.note_hz(63) - 1) > 1e-3      # ... where without the gap the correction glides from the last note's
    # the state survives the gap: a frame in the same hysteresis band after a gap keeps the previous target
    semis2 = np.concatenate([np.full(50, 61.0), np.full(10, np.nan), np.full(50, 61.6)])
    notes2 = []
    P.pitch_correct(_contour(semis2), HOP, 0, 0xfff, 440.0, 0.0, 1.0, notes=notes2)
    assert {n for _, n, _ in notes2} == {61}


def test_digital_silence():
    st = P.PitchStream(HOP, 0, 0xfff, 440.0, 50.0, 1.0)
    out = st.push(np.zeros(500))
    assert np.array_equal(out, np.zeros(500)) and st.meter == (0, 0.0, 0.0) and st.n_prev == P.NO_NOTE


@pytest.mark.parametrize('retune_ms', [20.0, 50.0, 150.0, 600.0])
def test_the_step_response_reaches_one_minus_1_over_e_after_retune_ms(retune_ms):
    # settled on 60.3 (c = -0.3), then the singer moves to exactly 62: d steps from -0.3 to 0
    m = round(retune_ms / HOP)
    semis = np.concatenate([np.full(4000, 60.3), np.full(m + 10, 62.0)])
    st = P.PitchStream(HOP, 0, 0xfff, 440.0, retune_ms, 1.0)
    c = []
    for f in _contour(semis):
        st.push([f])
        c.append(st.c)
    c0 = c[3999]
    assert abs(c0 + 0.3) < 1e-12
    reached = (c[3999 + m] - c0) / (0.0 - c0)
    assert abs(reached - (1 - math.exp(-1))) < 1e-9, reached


def test_the_meter():
    f0 = _contour(_gappy())
    st = P.PitchStream(HOP, 2, PITCH_SCALES['major'], 440.0, 40.0, 0.5)
    out = st.push(f0)
    v = f0 > 0
    applied = np.abs(12 * np.log2(out[v] / f0[v])) * 100
    n, mean, mx = st.meter
    assert n == int(v.sum()) and math.isclose(mean, applied.mean(), rel_tol=1e-9) and math.isclose(mx, applied.max(), rel_tol=1e-9)


def test_keys_and_scales():
    assert [pitch_key(k) for k in ('C', 'c#', 'Db', 'A', 'Bb', 'B', 7)] == [0, 1, 1, 9, 10, 11, 7]
    assert pitch_scale('major') == 0b101010110101 == P.SCALES['major'] and pitch_scale('Minor') == P.SCALES['minor']
    assert pitch_scale(0x123) == 0x123 and pitch_scale('chromatic') == 0xfff
    for bad in ('H', 'C##', ''):
        with pytest.raises(ValueError):
            pitch_key(bad)
    with pytest.raises(ValueError):
        pitch_scale('dorian')
    # the major scale's pitch classes in A: A B C# D E F# G#
    assert [(9 + j) % 12 for j in range(12) if PITCH_SCALES['major'] >> j & 1] == [9, 11, 1, 2, 4, 6, 8]


def test_pipeline_and_run_options():
    from realtime_yukarin_b200 import run
    from realtime_yukarin_b200.worker import pitch_settings
    assert pitch_settings({}) == dict(key=0, scale=0xfff, a4_hz=440.0, retune_ms=50.0, amount=1.0)
    assert pitch_settings(dict(key='Eb', scale='minor', retune_ms=0)) == dict(key=3, scale=P.SCALES['minor'], a4_hz=440.0,
                                                                              retune_ms=0.0, amount=1.0)
    for bad in (dict(key=12), dict(scale=0), dict(scale=0x1000), dict(a4_hz=390.0), dict(retune_ms=1500.0), dict(amount=1.5),
                dict(amount=math.nan), dict(speed=3)):
        with pytest.raises(ValueError):
            pitch_settings(bad)
    assert run.autotune_settings('A') == dict(key=9, scale=P.SCALES['major'], retune_ms=50.0, amount=1.0)
    assert run.autotune_settings('F#:minor', 0, 0.5) == dict(key=6, scale=P.SCALES['minor'], retune_ms=0.0, amount=0.5)
    assert run.autotune_settings('2:0x091')['scale'] == 0x091 and run.autotune_settings('C:chromatic')['scale'] == 0xfff
    args = run.make_parser().parse_args(['--config_path', 'c.yaml', '--autotune', 'Bb:major', '--retune_ms', '20', '--autotune_amount', '0.8'])
    assert (args.autotune, args.retune_ms, args.autotune_amount) == ('Bb:major', 20.0, 0.8)
    # refused before anything is loaded
    for kw in (dict(retune_ms=20.0), dict(autotune_amount=0.5), dict(autotune='H'), dict(autotune='C', autotune_amount=2.0),
               dict(autotune='C:dorian'), dict(load_state='x.state', autotune='C')):
        with pytest.raises(ValueError):
            run.run('does-not-exist.yaml', **kw)
