"""The clock drift stage and its controller without a GPU (DESIGN.md §4l): the FP64 oracle's properties, the controller against two
simulated sound cards, and RealtimePipeline / run.py over an oracle-backed stand-in engine."""
import math
from pathlib import Path

import numpy as np
import pytest
from scipy.signal import hilbert

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.drift import DriftController
from tests import drift_oracle as D
from tests import limiter_oracle as L
from tests.fake_engine import OracleEngine

W = D.W
FS = 24000
GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'


# ---- the prototype filter and the oracle ----
def test_the_filter_reads_whole_samples_exactly():
    T = wave_io.drift_filter()
    assert len(T) == 2 * W * D.P + 1 and T.dtype == np.float64
    whole = T[::D.P]
    assert whole[W] == 1.0 and np.count_nonzero(whole) == 1
    assert np.array_equal(T, T[::-1])                                   # symmetric about the centre


@pytest.mark.parametrize('seed', [0, 1])
def test_ppm_zero_is_a_pure_delay(seed):
    x = np.random.default_rng(seed).standard_normal(5000)
    assert D.inc_of(0.0) == 1 << 32
    y = D.resample(x, 0.0)
    assert np.array_equal(y, np.concatenate([np.zeros(W), x]))
    s = D.DriftStream(0.0)
    y = np.concatenate([s.push(x[:1234]), s.push(x[1234:1240]), s.push(x[1240:])])
    assert np.array_equal(y, np.concatenate([np.zeros(W), x])[:len(x)])


def _whole_signal(x, cuts, ppms, table):
    """outputs of a stream cut at `cuts` whose push j runs at ppms[j], from the absolute positions over the whole signal"""
    q, Q = 0, []
    for end, ppm in zip(cuts, ppms):
        inc = D.inc_of(ppm)
        while q < end * D.ONE:
            Q.append(q)
            q += inc
    b = np.concatenate([np.zeros(2 * W), x])
    return D.at_positions(b, np.array(Q, np.int64), table)


@pytest.mark.parametrize('seed', [3, 4, 5])
def test_any_cut_gives_the_whole_signal(seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(30000)
    sizes = list(rng.integers(0, 2500, 40))
    cuts = np.minimum(np.cumsum(sizes), len(x))
    ppms = list(rng.uniform(-1000, 1000, len(cuts)))
    s = D.DriftStream(ppms[0])
    out, a = [], 0
    for end, ppm in zip(cuts, ppms):
        s.set(ppm)                                                      # lands on the next push
        out.append(s.push(x[a:end]))
        a = end
    y = np.concatenate(out)
    assert np.array_equal(y, _whole_signal(x, cuts, ppms, s.table))
    assert (s.consumed, s.produced) == (cuts[-1], len(y))


@pytest.mark.parametrize('ppm', [-1000.0, -37.5, 12.3, 500.0])
def test_the_count_after_any_prefix_is_the_closed_form(ppm):
    rng = np.random.default_rng(7)
    s = D.DriftStream(ppm)
    inc = D.inc_of(ppm)
    for n in rng.integers(0, 3000, 50):
        s.push(np.zeros(n))
        assert s.produced == -(-s.consumed * D.ONE // inc)              # every m with m inc < N 2^32
        assert 0 <= s.pos < inc
        assert s.produced <= s.consumed + math.ceil(s.consumed * abs(ppm) * 1e-6) + 2


@pytest.mark.parametrize('ppm', [-500.0, 500.0])
def test_a_sine_comes_out_at_the_scaled_frequency(ppm):
    rate, f0 = 48000, 1000.0
    x = np.sin(2 * np.pi * f0 * np.arange(rate) / rate)
    y = D.resample(x, ppm)
    mid = y[4000:-4000]
    phase = np.unwrap(np.angle(hilbert(mid)))[2000:-2000]
    slope = np.polyfit(np.arange(len(phase)), phase, 1)[0]
    want = f0 / (1 + ppm * 1e-6)
    assert abs(slope * rate / (2 * np.pi) / want - 1) < 1e-7
    assert len(y) == -(-(len(x) + W) * D.ONE // D.inc_of(ppm))


@pytest.mark.parametrize('ppm', [-1000.0, -37.5, 12.3, 500.0, 1000.0])
def test_sines_up_to_035_fs_match_the_analytic_resampling(ppm):
    n = 20000
    inc = D.inc_of(ppm)
    for fr in (0.01, 0.1, 0.2, 0.3, 0.35):
        x = np.sin(2 * np.pi * fr * np.arange(n) + 0.3)
        y = D.resample(x, ppm)
        t = inc * np.arange(len(y), dtype=np.float64) / D.ONE - W       # each output's position in x
        ref = np.sin(2 * np.pi * fr * t + 0.3)
        sel = (t > 2 * W) & (t < n - 2 * W)
        snr = 10 * np.log10(np.sum(ref[sel] ** 2) / np.sum((y[sel] - ref[sel]) ** 2))
        assert snr >= 70.0, (fr, snr)


def test_inter_sample_peaks_of_limited_speech():
    """The limiter bounds the samples, not the waveform between them: resampling limited speech reads between the samples and can
    overshoot the ceiling.  The worst case over these trims on the golden speech, driven 6 dB into a -1 dB ceiling, is 0.317 dB."""
    x, fs = wave_io.read_wav(GOLDEN)
    x = x.astype(np.float64)
    g = 2.0 / np.abs(x).max()
    z = L.limit(x, fs, ceiling_db=-1.0, gain=g) * g
    c = 10 ** (-1 / 20)
    assert np.abs(z).max() <= c * (1 + 1e-12)
    over = {ppm: 20 * np.log10(np.abs(D.resample(z, ppm)).max() / c) for ppm in (-1000, -500, -37.5, 0, 12.3, 250, 500, 1000)}
    assert over[0] < 1e-12                                              # a pure delay reads the samples themselves
    assert round(max(over.values()), 3) == 0.317 and max(over, key=over.get) == 250


# ---- the controller against two simulated sound cards ----
def simulate(a_ppm, b_ppm, seed, control=True, hours=2.0, rate=48000, chunk=14400, cap_chunks=3, **kw):
    """The input card at rate (1 + a) paces the loop; each chunk goes through the drift stage into the output card's buffer, which
    drains at rate (1 + b) and starts with one chunk of silence.  The loop reads the buffer after each write, quantised down to 256
    frames and up to 5 ms late."""
    rng = np.random.default_rng(seed)
    a, b = a_ppm * 1e-6, b_ppm * 1e-6
    period = chunk / (rate * (1 + a))
    drain = rate * (1 + b) * period
    steps = int(hours * 3600 / period)
    ctl = DriftController(rate, chunk, **kw)
    pos, ppm = 0, 0.0
    inc = D.inc_of(ppm)
    fill, cap = float(chunk), cap_chunks * chunk
    fills, ppms = np.zeros(steps), np.zeros(steps)
    under = over = 0
    for k in range(steps):
        n = D.count(chunk, pos, inc)
        pos += n * inc - chunk * D.ONE
        fill += n
        if fill > cap:                                                  # the write blocks: the loop falls behind the input card
            over += 1
            fill = cap
        fills[k] = fill
        if control:
            ppm = ctl.update(math.floor((fill - rng.uniform(0, 0.005) * rate) / 256) * 256)
            inc = D.inc_of(ppm)
        ppms[k] = ppm
        fill -= drain
        if fill < 0:                                                    # the card ran dry: a glitch
            under += 1
            fill = 0.0
    return dict(fills=fills, ppms=ppms, under=under, over=over, per10=int(600 / period), setpoint=ctl.setpoint,
                truth=((1 + b) / (1 + a) - 1) * 1e6, slew=ctl.slew_ppm)


CLOCKS = [(250, -250), (-250, 250), (0, 100), (37, -12), (-400, 100), (120, 120), (-80, 300)]


@pytest.mark.parametrize('a,b', CLOCKS)
def test_the_controller_holds_the_output_buffer(a, b):
    r = simulate(a, b, seed=abs(31 * a + b))
    k = r['per10']
    assert r['under'] == 0 and r['over'] == 0
    assert np.max(np.abs(r['fills'][k:] - r['setpoint'])) < 14400      # within one chunk of the set-point after 10 minutes
    for j in range(1, len(r['ppms']) // k):
        assert abs(r['ppms'][j * k:(j + 1) * k].mean() - r['truth']) < 10.0, j
    assert np.max(np.abs(np.diff(r['ppms']))) <= r['slew'] + 1e-9
    assert np.max(np.abs(r['ppms'])) <= 500.0


@pytest.mark.parametrize('a,b', [c for c in CLOCKS if abs(c[0] - c[1]) >= 100])
def test_without_the_trim_the_buffer_runs_dry_or_over(a, b):
    r = simulate(a, b, seed=1, control=False)
    assert r['under'] > 0 or r['over'] > 0


def test_the_controller_state_round_trips():
    c = DriftController(48000, 14400, max_ppm=300.0)
    rng = np.random.default_rng(2)
    for v in rng.uniform(20000, 30000, 45):
        c.update(v)
    d = c.state()
    c2 = DriftController.from_state(d)
    for v in rng.uniform(20000, 30000, 20):
        assert c.update(v) == c2.update(v)
    assert c.state() == c2.state()
    with pytest.raises(ValueError):
        DriftController(48000, 14400, max_ppm=2500.0)


# ---- RealtimePipeline and run.py over the oracle-backed stand-in ----
class DriftEngine(OracleEngine):
    """OracleEngine with drift stages (tests/drift_oracle.py) and the session's echo far end recorded"""

    def drift_create(self, max_in, max_ppm=500.0, table=None):
        self.drifts = getattr(self, 'drifts', {})
        did = len(self.drifts)
        self.drifts[did] = dict(s=D.DriftStream(0.0, table), max_in=max_in, max_ppm=max_ppm, sets=[])
        return did

    def drift_set(self, did, ppm):
        R = self.drifts[did]
        assert abs(ppm) <= R['max_ppm']
        R['s'].set(ppm)
        R['sets'].append(ppm)

    def drift_get(self, did):
        s = self.drifts[did]['s']
        return s.ppm, s.inc

    def drift_push(self, did, x):
        assert len(x) <= self.drifts[did]['max_in']
        return self.drifts[did]['s'].push(np.asarray(x, np.float64))

    def drift_stats(self, did):
        s = self.drifts[did]['s']
        return s.consumed, s.produced

    def drift_destroy(self, did):
        self.drifts[did]['destroyed'] = True

    def session_echo_cancel(self, sid, taps=32, delay_ms=0.0):
        self.sessions[sid]['refs'] = []

    def session_set_echo_suppression(self, sid, db):
        pass

    def session_echo_reference(self, sid, far):
        self.sessions[sid]['refs'].append(np.array(far, np.float32))


def _config(small_models, **kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=0.1,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                           'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


def _run(small_models, steps, **kw):
    """(played chunks, far ends, drained chunks, engine) of a pipeline through run.audio_loop"""
    from realtime_yukarin_b200 import run
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models)
    n = cfg.in_audio_chunk
    x = synthetic.synthetic_speech((steps + 1) * 0.1, stream=43, silence_fraction=0.0)
    fake = DriftEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    pipe = RealtimePipeline(cfg, engine=fake, depth=1, **kw)
    pos, played = [0], []

    def read_chunk():
        a = pos[0]
        pos[0] += n
        return x[a:a + n] if a + n <= steps * n else None
    try:
        assert run.audio_loop(pipe, read_chunk, played.append) == steps
        drained = pipe.drain()
        refs = fake.sessions[pipe._sid].get('refs')
    finally:
        pipe.close()
    return played, refs, drained, fake


def test_the_pipeline_plays_the_drifted_stream_and_keeps_the_far_end(small_models):
    steps = 10
    plain, refs0, tail0, _ = _run(small_models, steps, echo_cancel=True)
    drifted, refs1, tail1, fake = _run(small_models, steps, echo_cancel=True, drift=250.0)
    assert any(np.any(p != 0) for p in plain), 'the stand-in played nothing: the check below would be empty'
    # the played stream is the drift of the stream the pipeline plays without it, and ends with the stage's W samples
    want = D.resample(np.concatenate(plain + tail0).astype(np.float64), 250.0).astype(np.float32)
    got = np.concatenate(drifted + tail1)
    assert got.dtype == np.float32 and np.array_equal(got, want)
    assert all(len(d) - len(p) in (0, 1) for d, p in zip(drifted, plain))        # 0.6 samples more per chunk at 250 ppm
    # the echo canceller's far end is the stream before the drift stage
    assert len(refs0) == len(refs1) == steps and all(np.array_equal(a, b) for a, b in zip(refs0, refs1))
    assert fake.drifts[0].get('destroyed')


def test_audio_loop_feeds_the_backlog_to_the_controller(small_models, monkeypatch):
    from realtime_yukarin_b200 import run
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models)
    fake = DriftEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    pipe = RealtimePipeline(cfg, engine=fake, depth=1, drift='auto', drift_max_ppm=300.0)
    seen = []
    monkeypatch.setattr(pipe._drift_ctl, 'update', lambda v: seen.append(v) or 7.5)
    readings = iter(range(100, 1000, 100))
    chunks = iter([np.zeros(cfg.in_audio_chunk, np.float32)] * 4)
    try:
        assert pipe.drift_auto
        assert run.audio_loop(pipe, lambda: next(chunks, None), lambda w: None, backlog=lambda: next(readings)) == 4
        assert seen == [100, 200, 300, 400] and fake.drifts[pipe._drift]['sets'] == [7.5] * 4
        assert pipe.drift_stats()['ppm'] == 7.5 and pipe.drift_stats()['auto']
        pipe.set_drift(-20.0)                                           # a fixed trim stops the controller
        assert not pipe.drift_auto and pipe.update_drift(5) == -20.0
    finally:
        pipe.close()


@pytest.mark.parametrize('kw', [dict(drift=600.0), dict(drift=float('nan')), dict(drift='on'), dict(drift='auto', drift_max_ppm=0.0),
                                dict(drift='auto', drift_max_ppm=2001.0), dict(drift=10.0, drift_max_ppm=5.0)])
def test_the_pipeline_refuses_bad_drift_settings_before_a_session_exists(small_models, kw):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = DriftEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    with pytest.raises(ValueError):
        RealtimePipeline(_config(small_models), engine=fake, **kw)
    assert not getattr(fake, 'sessions', None) and not getattr(fake, 'drifts', None)


def test_a_pipeline_without_drift_has_no_drift_stage(small_models):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = DriftEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    pipe = RealtimePipeline(_config(small_models), engine=fake)
    try:
        assert not getattr(fake, 'drifts', None) and not pipe.drift_auto and pipe.update_drift(100) is None
        with pytest.raises(RuntimeError, match='no drift stage'):
            pipe.drift_stats()
    finally:
        pipe.close()


def test_run_options(tmp_path):
    from realtime_yukarin_b200 import run
    p = run.make_parser()
    a = p.parse_args(['--config_path', 'cfg.yaml', '--drift'])
    assert a.drift == 500.0 and a.drift_ppm is None
    a = p.parse_args(['--config_path', 'cfg.yaml', '--drift', '800', '--drift_ppm', '12.5'])
    assert (a.drift, a.drift_ppm) == (800.0, 12.5)
    a = p.parse_args(['--config_path', 'cfg.yaml'])
    assert a.drift is None and a.drift_ppm is None
    with pytest.raises(ValueError, match='--drift needs live audio'):
        run.run(Path('does-not-exist.yaml'), wav_in=tmp_path / 'x.wav', drift=500.0)
    with pytest.raises(ValueError, match='exclude each other'):
        run.run(Path('does-not-exist.yaml'), drift=500.0, drift_ppm=10.0)
    for kw in (dict(drift=500.0), dict(drift_ppm=10.0)):
        with pytest.raises(ValueError, match='--load_state brings the stages'):
            run.run(Path('does-not-exist.yaml'), load_state=tmp_path / 'x.state', **kw)


def test_run_wav_mode_with_a_fixed_trim(tmp_path, small_models, monkeypatch):
    from realtime_yukarin_b200 import run
    cfg = _config(small_models)
    fakes = []

    class Converter:
        class acoustic_converter:
            class config:
                class dataset:
                    acoustic_param = None

    monkeypatch.setattr(run.Config, 'from_yaml', lambda path: cfg)
    monkeypatch.setattr(run.YukarinConverter, 'make_yukarin_converter', lambda **kw: Converter())
    n_in = 8 * cfg.in_audio_chunk
    x = synthetic.synthetic_speech(n_in / FS, stream=44, silence_fraction=0.0)[:n_in]
    monkeypatch.setattr(run.wave_io, 'load_wave', lambda *a, **kw: type('W', (), {'wave': x}))

    def engine():
        fakes.append(DriftEngine(small_models['stage1_model_path'], small_models['stage2_model_path']))
        return fakes[-1]
    lengths = {}
    for ppm in (None, 1000.0, -1000.0):
        out = tmp_path / f'{ppm}.wav'
        run.run(Path('cfg.yaml'), wav_in=tmp_path / 'in.wav', wav_out=out, engine=engine(), depth=1, drift_ppm=ppm)
        lengths[ppm] = len(wave_io.read_wav(out)[0])
    # (1 + ppm 1e-6) times the stream without drift followed by the stage's W samples, give or take one
    for ppm in (1000.0, -1000.0):
        assert abs(lengths[ppm] - (lengths[None] + W) * (1 + ppm * 1e-6)) <= 1.0
    assert fakes[1].drifts[0]['sets'] == [1000.0] and fakes[1].drifts[0]['max_ppm'] == 1000.0
