"""Host side of the per-session f0 map, without a GPU: the statistics file a measurement writes, the semitone arithmetic of
Engine.session_set_f0_map and the new run.py flags."""
import math
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import engine as eng
from realtime_yukarin_b200 import models, run, synthetic


def test_statistics_file_round_trips(tmp_path):
    """write_f0_statistics writes what F0Converter reads and what upstream's readers do with numpy.load(...).item(); the suffix is
    kept as given."""
    mean, var = 5.1234567890123, 0.0321
    for name in ('input_statistics.npy', 'measured.stats'):
        path = tmp_path / name
        models.write_f0_statistics(path, mean, var)
        assert path.exists() and sorted(p.name for p in tmp_path.iterdir() if p.name.startswith(path.stem)) == [name]
        d = np.load(str(path), allow_pickle=True).item()
        assert set(d) == {'mean', 'var'} and d['mean'] == mean and d['var'] == var
    target = synthetic.write_synthetic_models(tmp_path / 'm', seed=1, base1=16, base2=16)['target_statistics_path']
    f0c = models.F0Converter(tmp_path / 'input_statistics.npy', target)
    assert f0c.input_mean == mean and f0c.input_var == var
    assert f0c.stats()[:2] == (mean, math.sqrt(var))


@pytest.mark.parametrize('mean,var', [(float('nan'), 0.04), (5.0, 0.0), (5.0, -1.0), (5.0, float('inf'))])
def test_statistics_file_rejects_unusable_values(tmp_path, mean, var):
    with pytest.raises(ValueError):
        models.write_f0_statistics(tmp_path / 's.npy', mean, var)
    assert not (tmp_path / 's.npy').exists()


def test_semitones_move_the_target_mean_only():
    cur = dict(in_mean=5.0, in_std=0.2, target_mean=5.5, target_std=0.25)
    assert eng.updated_f0_map(cur) == cur
    up = eng.updated_f0_map(cur, semitones=12)
    assert up['target_mean'] == 5.5 + math.log(2.0) and {k: up[k] for k in ('in_mean', 'in_std', 'target_std')} == \
        {k: cur[k] for k in ('in_mean', 'in_std', 'target_std')}
    # an octave doubles f0 whatever the input: exp((x - mu_i) / sd_i * sd_t + mu_t + ln 2) = 2 exp(...)
    x = math.log(180.0)
    f = lambda m: math.exp((x - m['in_mean']) / m['in_std'] * m['target_std'] + m['target_mean'])
    assert f(up) == pytest.approx(2.0 * f(cur), rel=1e-14)
    assert f(eng.updated_f0_map(cur, semitones=-1)) == pytest.approx(f(cur) * 2.0 ** (-1.0 / 12.0), rel=1e-14)
    # given values replace, None keeps, and the shift applies to the target mean that was given
    new = eng.updated_f0_map(cur, in_mean=4.8, target_mean=5.0, semitones=3)
    assert new == dict(in_mean=4.8, in_std=0.2, target_mean=5.0 + 3 * math.log(2.0) / 12.0, target_std=0.25)
    assert cur['target_mean'] == 5.5                       # the argument is not modified


def test_run_flags():
    p = run.make_parser()
    a = p.parse_args([])
    assert a.measure_input_statistics is None and a.follow_input_f0 is None and a.pitch == 0.0
    a = p.parse_args(['--wav_in', 'a.wav', '--measure_input_statistics', 'out.npy'])
    assert a.measure_input_statistics == Path('out.npy') and a.wav_in == Path('a.wav') and a.follow_input_f0 is None
    assert p.parse_args(['--follow_input_f0']).follow_input_f0 == 200
    a = p.parse_args(['--follow_input_f0', '50', '--pitch', '-2.5'])
    assert a.follow_input_f0 == 50 and a.pitch == -2.5
    with pytest.raises(SystemExit):
        p.parse_args(['--pitch', 'high'])


def test_measured_statistics_are_saved_only_when_usable(tmp_path, capsys):
    class Pipe:
        def __init__(self, triple):
            self.triple = triple

        def measured_f0(self):
            return self.triple

    out = tmp_path / 'stats.npy'
    assert run.save_measured_statistics(Pipe((0, 0.0, 0.0)), out) is False and not out.exists()
    assert run.save_measured_statistics(Pipe((500, 5.0, 0.0)), out) is False and not out.exists()
    assert run.save_measured_statistics(Pipe((500, math.log(200.0), 0.2)), out) is True
    d = np.load(str(out), allow_pickle=True).item()
    assert d['mean'] == math.log(200.0) and d['var'] == 0.2 * 0.2
    text = capsys.readouterr().out
    assert '500 voiced frames' in text and '200.0 Hz' in text
