"""The FP64 reference of the output limiter (DESIGN.md DECIDE L1-L4) and its host options, without a GPU:
  * a stream cut into steps of any size is bitwise the whole signal, delayed by L;
  * |G z| never exceeds the ceiling, on impulses, a clipped sine and scaled golden speech;
  * below the ceiling the output is y bit for bit;
  * a lone peak lowers the gain on exactly [p - L + 1, p + R + L - 1], down and back up in linear ramps;
  * a setting change applies to the samples of the step that brings it;
  * RealtimePipeline and run.py hand the options through and refuse bad ones before a session exists.
"""
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io

from . import limiter_oracle as LO
from .fake_engine import OracleEngine

FS = 24000
GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
SHAPES = [(24000, 5.0, 50.0), (48000, 10.0, 500.0), (24000, 0.5, 0.0), (44100, 2.5, 7.0)]


def _golden():
    x, fs = wave_io.read_wav(GOLDEN)
    assert fs == FS
    return np.asarray(x, np.float64)


def _bound_holds(z, db, gain):
    return np.all(np.abs(gain * z) <= LO.ceiling(db) * (1 + 1e-12))


@pytest.mark.parametrize('rate,la,hold', SHAPES)
def test_steps_of_any_size_are_the_whole_signal(rate, la, hold):
    rng = np.random.default_rng(rate + int(hold))
    y = _golden()[:30000] * 3.0
    st = LO.LimiterStream(rate, la, hold)
    st.set(-3.0, 1.5)
    outs, a = [], 0
    while a < len(y):
        n = int(rng.choice([0, 1, 7, 480, 2047, 7200, 14400]))
        outs.append(st.push(y[a:a + n]))
        a += n
    got = np.concatenate(outs)[:len(y)]
    want = np.concatenate([np.zeros(st.L), LO.limit(y, rate, la, hold, -3.0, 1.5)])[:len(y)]
    assert np.array_equal(got, want)
    assert np.count_nonzero(want != np.concatenate([np.zeros(st.L), y])[:len(y)]) > 100, 'the limiter never engaged'


def _signals():
    rng = np.random.default_rng(5)
    imp = rng.normal(0, 0.02, 24000)
    imp[rng.integers(0, 24000, 40)] = rng.uniform(-4, 4, 40)
    t = np.arange(24000) / FS
    sine = np.clip(3.0 * np.sin(2 * np.pi * 220 * t), -2.0, 2.0)
    return {'impulses': imp, 'clipped_sine': sine, 'speech_x8': 8.0 * _golden()}


@pytest.mark.parametrize('name', ['impulses', 'clipped_sine', 'speech_x8'])
@pytest.mark.parametrize('db,gain', [(-1.0, 1.0), (-6.0, 2.0), (-24.0, 0.5), (0.0, 3.0)])
def test_the_played_level_stays_under_the_ceiling(name, db, gain):
    y = _signals()[name]
    for rate, la, hold in SHAPES[:3]:
        z = LO.limit(y, rate, la, hold, db, gain)
        assert _bound_holds(z, db, gain), (rate, la, hold)
        assert np.max(np.abs(gain * y)) > LO.ceiling(db)


def test_below_the_ceiling_the_output_is_the_input_bit_for_bit():
    y = _golden()
    y = y * (0.8 / np.max(np.abs(y)))
    for rate, la, hold in SHAPES:
        z, g = LO.limit(y, rate, la, hold, -1.0, 1.0, return_gain=True)
        assert np.all(g == 1.0) and np.array_equal(z, y)
        st = LO.LimiterStream(rate, la, hold)
        out = np.concatenate([st.push(y[a:a + 3000]) for a in range(0, len(y), 3000)])
        assert np.array_equal(out[st.L:], y[:len(y) - st.L]) and not np.any(out[:st.L])


@pytest.mark.parametrize('rate,la,hold', SHAPES)
def test_a_lone_peak_lowers_the_gain_on_exactly_its_support(rate, la, hold):
    L, R = LO.shape(rate, la, hold)
    n, p = 60000, 20000
    y = np.full(n, 0.1)
    y[p] = 2.0
    z, g = LO.limit(y, rate, la, hold, -1.0, 1.0, return_gain=True)
    idx = np.flatnonzero(g < 1.0)
    assert idx[0] == p - L + 1 and idx[-1] == p + R + L - 1 and len(idx) == R + 2 * L - 1
    g0 = LO.ceiling(-1.0) / 2.0
    assert g[p] <= g0 * (1 + 1e-12) and abs(g[p] - g0) < 1e-12
    down, hold_part, up = g[p - L + 1:p + 1], g[p:p + R + 1], g[p + R:p + R + L]
    assert np.all(np.diff(down) < 0) and np.all(np.diff(up) > 0)
    assert np.allclose(hold_part, g0, rtol=1e-12, atol=0)
    # linear ramps: steps of (1 - g0) / L
    assert np.allclose(np.diff(down), -(1 - g0) / L, rtol=1e-9, atol=1e-15)
    assert abs(z[p]) * 1.0 <= LO.ceiling(-1.0) * (1 + 1e-12)


def test_a_setting_change_applies_from_the_samples_of_its_step():
    y = 4.0 * _golden()[:40000]
    rate, la, hold = 24000, 5.0, 20.0
    st = LO.LimiterStream(rate, la, hold)
    steps = [7200] * 5 + [4000]
    cdb, gains, outs, a = [], [], [], 0
    for k, n in enumerate(steps):
        db, gain = (-1.0, 1.0) if k < 2 else (-9.0, 2.0) if k < 4 else (-0.5, 0.7)
        st.set(db, gain)
        outs.append(st.push(y[a:a + n]))
        cdb += [db] * n
        gains += [gain] * n
        a += n
    got = np.concatenate(outs)
    want = np.concatenate([np.zeros(st.L), LO.limit(y[:a], rate, la, hold, np.array(cdb), np.array(gains))])[:a]
    assert np.array_equal(got, want)
    # the change reaches g of the L - 1 samples before the step's first one (their look-ahead): with the delay of L, no output before
    # index 2 * 7200 + 1 differs from the run without the change
    const = np.concatenate([np.zeros(st.L), LO.limit(y[:a], rate, la, hold, -1.0, 1.0)])[:a]
    first = np.flatnonzero(got != const)[0]
    assert 2 * 7200 + 1 <= first < 2 * 7200 + 2000


def test_the_meter_counts_the_limited_samples_of_the_last_step():
    y = 5.0 * _golden()[:24000]
    st = LO.LimiterStream(24000, 5.0, 50.0)
    outs = [st.push(y[a:a + 7200]) for a in range(0, 21600, 7200)]
    z, g = LO.limit(y, 24000, 5.0, 50.0, -1.0, 1.0, return_gain=True)
    gl = g[14400 - st.L:21600 - st.L]
    assert st.last_meter == LO.meter(gl) and st.last_meter[1] > 0
    assert np.isclose(st.last_meter[0], -20 * np.log10(gl.min()))


# ---- RealtimePipeline and run.py over the oracle-backed stand-in ----
class LimiterEngine(OracleEngine):
    """OracleEngine with the session's output limiter (LimiterStream) after StreamOracle"""

    def session_limiter(self, sid, lookahead_ms=5.0, hold_ms=50.0):
        self.sessions[sid]['lim'] = LO.LimiterStream(FS, lookahead_ms, hold_ms)
        self.sessions[sid]['lim_settings'] = []

    def session_set_limiter(self, sid, ceiling_db, gain=1.0):
        self.sessions[sid]['lim'].set(ceiling_db, gain)
        self.sessions[sid]['lim_settings'].append((ceiling_db, gain))

    def session_limiter_stats(self, sid):
        return self.sessions[sid]['lim'].last_meter

    def session_submit(self, sid, wave):
        t = super().session_submit(sid, wave)
        S = self.sessions[sid]
        if 'lim' in S:
            S['last'] = S['lim'].push(S['last'])
            S['out'][t] = S['last']
        return t


def _config(small_models, **kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=0.1,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                           'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


def _play(small_models, scale, **kw):
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models, output_scale=scale)
    fake = LimiterEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    n, steps = cfg.in_audio_chunk, 16
    x = synthetic.synthetic_speech((steps + 1) * 0.1, stream=31, silence_fraction=0.0)
    pipe = RealtimePipeline(cfg, engine=fake, **kw)
    try:
        played = [pipe.process(x[k * n:(k + 1) * n], block=True) for k in range(steps)]
        played += pipe.drain()
        S = fake.sessions[pipe._sid]
        stats = pipe.limiter_stats() if 'lim' in S else None
        settings = list(S.get('lim_settings', []))
        if 'lim' in S:
            pipe.set_limiter(-6.0)
            settings = list(S['lim_settings'])
    finally:
        pipe.close()
    return np.concatenate(played), settings, stats


def test_the_pipeline_plays_under_the_ceiling_only_with_the_limiter(small_models):
    plain, _, _ = _play(small_models, 60.0)
    assert np.max(np.abs(plain)) > LO.ceiling(-1.0), 'the stand-in never crossed the ceiling: the check below would be empty'
    played, settings, stats = _play(small_models, 60.0, limiter=-1.0, limiter_lookahead_ms=2.0, limiter_hold_ms=10.0)
    # the host still multiplies by output_scale; the float32 cast adds at most half an ulp
    assert np.max(np.abs(played)) <= LO.ceiling(-1.0) * (1 + 2 ** -23)
    assert settings == [(-1.0, 60.0), (-6.0, 60.0)]
    assert stats[1] >= 0


@pytest.mark.parametrize('kw', [dict(limiter=1.0), dict(limiter=-30.0), dict(limiter=float('nan')), dict(limiter=-1.0, limiter_lookahead_ms=0.2),
                                dict(limiter=-1.0, limiter_lookahead_ms=11.0), dict(limiter=-1.0, limiter_hold_ms=-1.0),
                                dict(limiter=-1.0, limiter_hold_ms=600.0)])
def test_the_pipeline_refuses_bad_limiter_settings_before_a_session_exists(small_models, kw):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = LimiterEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    with pytest.raises(ValueError):
        RealtimePipeline(_config(small_models), engine=fake, **kw)
    assert not getattr(fake, 'sessions', None)


def test_the_pipeline_refuses_the_limiter_with_a_non_positive_output_scale(small_models):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = LimiterEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    with pytest.raises(ValueError):
        RealtimePipeline(_config(small_models, output_scale=0.0), engine=fake, limiter=-1.0)


def test_run_options():
    from realtime_yukarin_b200 import run
    p = run.make_parser()
    a = p.parse_args(['--config_path', 'cfg.yaml', '--limit'])
    assert a.limit == -1.0 and a.limit_lookahead is None and a.limit_hold is None
    a = p.parse_args(['--config_path', 'cfg.yaml', '--limit', '-3', '--limit_lookahead', '2.5', '--limit_hold', '100'])
    assert (a.limit, a.limit_lookahead, a.limit_hold) == (-3.0, 2.5, 100.0)
    assert p.parse_args(['--config_path', 'cfg.yaml']).limit is None
    for kw in (dict(limit_lookahead=2.0), dict(limit_hold=10.0)):
        with pytest.raises(ValueError, match='need --limit'):
            run.run(Path('does-not-exist.yaml'), **kw)
