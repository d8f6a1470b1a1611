"""The FP64 reference of the automatic gain control (DESIGN.md DECIDE A1-A4) and its host options, without a GPU:
  * a stream cut into steps of any size, steps shorter than one block included, is bitwise the whole signal;
  * max_gain_db = 0, and an input wholly under the gate, return x bit for bit;
  * the gain stays within [1 / gmax, gmax] and moves by at most the slew factors from block to block;
  * scaled golden speech converges to the target; the gain holds through the pauses of synthetic speech;
  * a setting change applies from the first block whose last sample its step brings; the meter is the recursion's;
  * RealtimePipeline and run.py hand the options through and refuse bad ones before a session exists.
"""
import math
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io

from . import agc_oracle as A
from .fake_engine import OracleEngine

FS = 24000
GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
SETTINGS = [(-26.0, 20.0, -50.0), (-12.0, 6.0, -30.0), (-40.0, 30.0, -80.0), (-6.0, 10.0, -20.0)]


def _golden(seconds=4.0, db=0.0):
    x, fs = wave_io.read_wav(GOLDEN)
    assert fs == FS
    x = np.tile(np.asarray(x, np.float64), int(np.ceil(seconds * FS / len(x))))[:round(seconds * FS)]
    return (x * 10 ** (db / 20)).astype(np.float32)


@pytest.mark.parametrize('fs', [24000, 48000])
@pytest.mark.parametrize('settings', SETTINGS)
def test_steps_of_any_size_are_the_whole_signal(fs, settings):
    rng = np.random.default_rng(fs + int(settings[0]))
    x = _golden(6.0, db=-6.0)
    want = A.agc(x, fs, *settings)
    st = A.AgcStream(fs, *settings)
    outs, a = [], 0
    while a < len(x):
        n = int(rng.choice([0, 1, 7, 255, 256, 257, 511, 7200, 14400]))
        outs.append(st.push(x[a:a + n]))
        a += n
    assert np.array_equal(np.concatenate(outs), want)
    assert not np.array_equal(want, x), 'the gain never moved'


def test_no_gain_and_input_under_the_gate_return_x_bit_for_bit():
    x = _golden(3.0, db=-20.0)
    for fs in (24000, 48000):
        assert np.array_equal(A.agc(x, fs, -26.0, 0.0, -50.0), x)
        st = A.AgcStream(fs, -26.0, 0.0, -50.0)
        assert np.array_equal(np.concatenate([st.push(x[a:a + 1000]) for a in range(0, len(x), 1000)]), x)
    # the golden speech at -60 dB sits wholly under a gate of -50 dB: no block is active, the level never starts
    quiet = _golden(3.0, db=-60.0)
    assert A.level_db(quiet) < -70.0
    z, g, active = A.agc(quiet, FS, return_gain=True)
    assert not active.any() and np.all(g == 1.0) and np.array_equal(z, quiet)


@pytest.mark.parametrize('settings', SETTINGS)
def test_the_gain_stays_bounded_and_slews(settings):
    target_db, max_gain_db, gate_db = settings
    P = A.params(FS, *settings)
    for db in (-40.0, -20.0, 0.0, 10.0):
        x = np.clip(_golden(8.0, db=db), -8.0, 8.0)
        _, g, active = A.agc(x, FS, *settings, return_gain=True)
        assert np.all(g >= P['ginv']) and np.all(g <= P['gmax'])
        prev = np.concatenate([[1.0], g[:-1]])
        assert np.all(g <= prev * P['s_up']) and np.all(g >= prev * P['s_dn'])
        assert np.all(g[~active] == prev[~active])
    # the slew in dB per second: 6 up, 24 down
    assert math.isclose(20 * math.log10(P['s_up']) * FS / A.B, 6.0, rel_tol=1e-12)
    assert math.isclose(20 * math.log10(P['s_dn']) * FS / A.B, -24.0, rel_tol=1e-12)


# Tolerance of the convergence test, from the oracle on the golden recording looped to 16 s: the active blocks of the second half come
# out at -26.00 dB at -20 dB and 0 dB (within 0.01 dB: E smooths over 0.4 s, so the output level rides the speech's own syllable-scale
# variation around the target) and at -25.16 dB at +10 dB, where the recording (-5.2 dB) needs more than the 20 dB cap of attenuation.
@pytest.mark.parametrize('db, want', [(-20.0, -26.0), (0.0, -26.0), (10.0, -25.16)])
def test_scaled_golden_speech_converges_to_the_target(db, want):
    x = _golden(16.0, db=db)
    z, g, active = A.agc(x, FS, return_gain=True)
    nb = len(g)
    blocks = z[:nb * A.B].astype(np.float64).reshape(nb, A.B)
    half = np.arange(nb) >= nb // 2
    got = 10 * math.log10(float(np.mean(blocks[half & active] ** 2)))
    print(f'input at {db:+.0f} dB (level {A.level_db(x):.2f} dB): active output level of the second half {got:.2f} dB, '
          f'gain {20 * math.log10(g[-1]):+.2f} dB')
    assert abs(got - want) < 0.05
    if db == -20.0:        # +6 dB/s up: +8.5 dB after 2 s, the final +10 dB after 4 s
        assert 8.0 < 20 * math.log10(g[round(2 * FS / A.B)]) < 9.0
        assert 20 * math.log10(g[round(4 * FS / A.B)]) > 9.9


def test_the_gain_holds_through_the_pauses_of_synthetic_speech():
    x = synthetic.synthetic_speech(12.0, stream=3).astype(np.float32)
    _, g, active = A.agc(x, FS, return_gain=True)
    assert active.sum() > 0.6 * len(g) and (~active).sum() > 0.1 * len(g)
    prev = np.concatenate([[1.0], g[:-1]])
    assert np.all(g[~active] == prev[~active])
    # every pause of at least ten blocks (its noise 40 dB under the speech, under the gate) leaves the gain where the speech left it
    runs = np.flatnonzero(np.diff(np.concatenate([[0], (~active).astype(int), [0]])))
    pauses = [(a, b) for a, b in zip(runs[::2], runs[1::2]) if b - a >= 10 and a > 0]
    assert pauses
    for a, b in pauses:
        assert np.all(g[a:b] == g[a - 1])
    steps_db = np.abs(np.diff(20 * np.log10(np.concatenate([[1.0], g]))))
    assert steps_db.max() <= 24.0 * A.B / FS + 1e-9


def test_a_setting_change_applies_from_the_first_block_its_step_completes():
    x = _golden(6.0, db=-10.0)
    steps = [7200] * 10 + [len(x) - 72000]
    change = {4: (-12.0, 20.0, -50.0), 7: (-30.0, 6.0, -40.0)}
    st = A.AgcStream(FS)
    outs, a, per_block = [], 0, []
    settings = (-26.0, 20.0, -50.0)
    for k, n in enumerate(steps):
        if k in change:
            settings = change[k]
            st.set(*settings)
        outs.append(st.push(x[a:a + n]))
        a += n
        per_block += [settings] * ((a // A.B) - len(per_block))     # the blocks whose last sample this step brought
    cols = np.array(per_block).T
    want = A.agc(x, FS, cols[0], cols[1], cols[2])
    assert np.array_equal(np.concatenate(outs), want)
    # the first sample that differs from the run without changes lies in the block after the first one the change applied to
    const = A.agc(x, FS)
    first = int(np.flatnonzero(np.concatenate(outs) != const)[0])
    m = 4 * 7200 // A.B                                              # the first block completed by step 4: it holds its first sample
    assert (m + 1) * A.B <= first < (m + 40) * A.B


def test_the_meter_is_the_recursions_last_step():
    x = _golden(4.0, db=-20.0)
    st = A.AgcStream(FS)
    assert st.last_meter == (-math.inf, 0.0, 0)
    for a in range(0, 3 * 7200, 7200):
        st.push(x[a:a + 7200])
    _, g, active = A.agc(x[:3 * 7200], FS, return_gain=True)
    level, gain_db, n = st.last_meter
    assert n == int(active[2 * 7200 // A.B:].sum()) and n > 0
    assert gain_db == 20 * math.log10(g[-1])
    assert level == 10 * math.log10(st.E) and -40.0 < level < -30.0
    quiet = A.AgcStream(FS)
    quiet.push(_golden(0.3, db=-70.0))
    assert quiet.last_meter == (-math.inf, 0.0, 0)


# ---- RealtimePipeline and run.py over the oracle-backed stand-in ----
class AgcEngine(OracleEngine):
    """OracleEngine with the session's gain control (AgcStream) in front of StreamOracle"""

    def session_agc(self, sid, target_db=-26.0, max_gain_db=20.0, gate_db=-50.0):
        self.sessions[sid]['agc'] = A.AgcStream(FS, target_db, max_gain_db, gate_db)
        self.sessions[sid]['agc_settings'] = [(target_db, max_gain_db, gate_db)]
        self.sessions[sid]['agc_in'] = []

    def session_get_agc(self, sid):
        t, m, g = self.sessions[sid]['agc_settings'][-1]
        return dict(target_db=t, max_gain_db=m, gate_db=g, linear=A.params(FS, t, m, g))

    def session_set_agc(self, sid, target_db=None, max_gain_db=None, gate_db=None):
        cur = self.session_get_agc(sid)
        s = (cur['target_db'] if target_db is None else target_db, cur['max_gain_db'] if max_gain_db is None else max_gain_db,
             cur['gate_db'] if gate_db is None else gate_db)
        self.sessions[sid]['agc'].set(*s)
        self.sessions[sid]['agc_settings'].append(s)

    def session_agc_stats(self, sid):
        return self.sessions[sid]['agc'].last_meter

    def session_submit(self, sid, wave):
        S = self.sessions[sid]
        if 'agc' in S:
            S['agc_in'].append(np.asarray(wave, np.float32).copy())
            wave = S['agc'].push(wave)
        return super().session_submit(sid, wave)


def _config(small_models, **kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=0.1,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                           'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


def test_the_pipeline_controls_the_scaled_input(small_models):
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models, input_scale=0.125)
    fake = AgcEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    n, steps = cfg.in_audio_chunk, 12
    x = synthetic.synthetic_speech((steps + 1) * 0.1, stream=41).astype(np.float32)
    pipe = RealtimePipeline(cfg, engine=fake, agc=-20.0, agc_max_gain_db=12.0, agc_gate_db=-60.0)
    try:
        for k in range(steps):
            pipe.process(x[k * n:(k + 1) * n], block=True)
        S = fake.sessions[pipe._sid]
        stats = pipe.agc_stats()
        pipe.set_agc(gate_db=-45.0)
        settings = list(S['agc_settings'])
        fed = np.concatenate(S['agc_in'])
    finally:
        pipe.close()
    # the gain control sees the chunks after input_scale
    assert np.array_equal(fed, np.concatenate([x[k * n:(k + 1) * n] * np.float32(0.125) for k in range(steps)]))
    assert settings == [(-20.0, 12.0, -60.0), (-20.0, 12.0, -45.0)]
    assert stats[2] >= 0 and stats[0] > -60.0


@pytest.mark.parametrize('kw', [dict(agc=-5.0), dict(agc=-41.0), dict(agc=float('nan')), dict(agc=-26.0, agc_max_gain_db=-1.0),
                                dict(agc=-26.0, agc_max_gain_db=31.0), dict(agc=-26.0, agc_gate_db=-10.0),
                                dict(agc=-26.0, agc_gate_db=-90.0), dict(agc=-26.0, agc_gate_db=float('inf'))])
def test_the_pipeline_refuses_bad_agc_settings_before_a_session_exists(small_models, kw):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = AgcEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    with pytest.raises(ValueError):
        RealtimePipeline(_config(small_models), engine=fake, **kw)
    assert not getattr(fake, 'sessions', None)


def test_run_options():
    from realtime_yukarin_b200 import run
    p = run.make_parser()
    a = p.parse_args(['--config_path', 'cfg.yaml', '--agc'])
    assert a.agc == -26.0 and a.agc_max_gain is None and a.agc_gate is None
    a = p.parse_args(['--config_path', 'cfg.yaml', '--agc', '-20', '--agc_max_gain', '12', '--agc_gate', '-60'])
    assert (a.agc, a.agc_max_gain, a.agc_gate) == (-20.0, 12.0, -60.0)
    assert p.parse_args(['--config_path', 'cfg.yaml']).agc is None
    for kw in (dict(agc_max_gain=10.0), dict(agc_gate=-40.0)):
        with pytest.raises(ValueError, match='need --agc'):
            run.run(Path('does-not-exist.yaml'), **kw)
