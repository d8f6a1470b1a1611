"""The automatic gain control of a streaming session (ryk_session_agc and its calls) and the whole-signal ryk_agc, at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models.

  * ryk_agc is the FP64 oracle (tests/agc_oracle.py) bit for bit at 24 and 48 kHz over levels, settings and signals with pauses and
    bursts, and the linear values a session uses are the oracle's;
  * a session with the AGC is bitwise a session without it fed ryk_agc of what it analyses: at 24 kHz, at a 48 kHz input rate, with
    noise suppression and echo cancellation on in both enabling orders, through push, submit / collect and push_device;
  * a setting change made with chunks in flight lands on the next submitted step; group members are the session alone; a voice
    switch keeps the AGC's state; the meter is the oracle's;
  * one kernel per step and none for other sessions; refusals change nothing; cycles return memory; run.py --agc is the pipeline's.
"""
import math
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import AGC_LINEAR, RykError

from . import agc_oracle as A
from . import denoise_oracle as DO
from . import echo_oracle as E
from .test_gpu_f0_control import (EXTRA, FS, N, T, _cfg, _new_voice, _push, _same, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_launch_count import _run_child, _window
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
QUIET_DB = -18.0              # the speech of the session tests sits this far under its recorded level: the AGC lifts it by ~7 dB


def _golden(seconds, db=0.0):
    x, rate = wave_io.read_wav(GOLDEN)
    assert rate == FS
    x = np.tile(np.asarray(x, np.float64), int(np.ceil(seconds * FS / len(x))))[:round(seconds * FS)]
    return (x * 10 ** (db / 20)).astype(np.float32)


def _speech(seconds, stream, db=QUIET_DB):
    """synthetic speech (with its pauses) scaled to db under its own level"""
    return (synthetic.synthetic_speech(seconds, stream=stream) * 10 ** (db / 20)).astype(np.float32)


def _chunks(x, n=N):
    return [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(len(x) // n)]


def _agc_session(engine, made, settings=(-26.0, 20.0, -50.0), voice=0):
    sid = made.create(voice=voice)
    engine.session_agc(sid, *settings)
    return sid


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_the_whole_signal_call_is_the_oracle(engine):
    rng = np.random.default_rng(5)
    bursts = np.zeros(round(6.0 * FS), np.float32)
    for a in rng.integers(0, len(bursts) - 4000, 12):
        bursts[a:a + 4000] += rng.normal(0, 0.3, 4000).astype(np.float32)
    signals = {'golden': _golden(16.0), 'speech': _speech(6.0, 1, 0.0), 'bursts': bursts}
    cases = 0
    for fs in (24000, 48000):
        for name, x in signals.items():
            for db in (-30.0, -10.0, 6.0):
                y = (x * np.float32(10 ** (db / 20))).astype(np.float32)
                for settings in ((-26.0, 20.0, -50.0), (-12.0, 6.0, -30.0), (-40.0, 30.0, -80.0), (-20.0, 0.0, -50.0)):
                    got = engine.agc(y, fs, *settings)
                    want = A.agc(y, fs, *settings)
                    assert np.array_equal(got, want), (fs, name, db, settings, int(np.count_nonzero(got != want)))
                    cases += 1
    print(f'ryk_agc is the FP64 oracle bit for bit in {cases} cases (the 16 s signal runs in two pieces)')
    x = signals['golden'][:N]
    assert np.array_equal(engine.agc(x, FS, -26.0, 0.0, -50.0), x)


def test_the_linear_values_are_the_oracles(engine, made):
    sid = _agc_session(engine, made, (-30.0, 12.0, -55.0))
    got = engine.session_get_agc(sid)
    assert (got['target_db'], got['max_gain_db'], got['gate_db']) == (-30.0, 12.0, -55.0)
    assert got['linear'] == A.params(FS, -30.0, 12.0, -55.0) and tuple(got['linear']) == AGC_LINEAR == A.NAMES
    engine.session_set_agc(sid, max_gain_db=25.0)
    assert engine.session_get_agc(sid)['linear'] == A.params(FS, -30.0, 25.0, -55.0)


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rate', [FS, 48000])
def test_the_stream_is_the_whole_signal_bitwise(engine, made, rate):
    steps = 24
    x24 = _speech((steps + 1) * T, stream=1001)
    a = made.create()
    if rate != FS:
        engine.session_set_input_rate(a, rate)
    engine.session_agc(a)
    geo = engine.session_io_geometry(a)
    c = made.create()
    if rate != FS:
        engine.session_set_input_rate(c, rate)
    assert geo == engine.session_io_geometry(c), 'the AGC changes no geometry'
    if rate == FS:
        x, model = x24, x24
    else:
        x = wave_io.resample(x24, FS, rate, engine)
        d_rs = geo['delay_in']
        assert d_rs == wave_io.stream_input_geometry(rate, FS, T)[2]
        model = np.concatenate([np.zeros(d_rs, np.float32), engine.resample_poly(x, 1, 2, wave_io.resample_filter(1, 2))])
    ref_in = engine.agc(model[:steps * N], FS)
    assert not np.array_equal(ref_in, model[:steps * N])
    out_a = _push(engine, a, _chunks(x, geo['n_in'])[:steps])
    out_b = _push(engine, made.create(), _chunks(ref_in)[:steps])
    assert sum(len(o) for o in out_a) > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert _same(out_a, out_b)
    level, gain, active = engine.session_agc_stats(a)
    print(f'rate {rate}: level {level:.2f} dB, gain {gain:+.2f} dB, {active} active blocks in the last step')
    assert gain > 3.0


@pytest.mark.parametrize('order', ['agc', 'frame stage'])
def test_with_noise_suppression_and_echo_cancellation_it_controls_the_frame_stages_output(engine, made, order):
    steps = 20
    far = _golden((steps + 1) * T, db=-6.0)
    echo = E.echo_of(far, E.room_ir(30, seed=1011))
    near = _speech((steps + 1) * T, stream=1011, db=-12.0)
    mic = (echo + near[:len(echo)]).astype(np.float32)
    phi = DO.frame_powers(mic, 3, 60).mean(axis=0)
    a = made.create()
    calls = [lambda: engine.session_agc(a), lambda: engine.session_echo_cancel(a, taps=32), lambda: engine.session_denoise(a)]
    for c in (calls if order == 'agc' else calls[1:] + calls[:1]):
        c()
    engine.session_set_noise_profile(a, phi)
    assert engine.session_io_geometry(a)['delay_in'] == DO.D
    stage = engine.echo_cancel(mic[:steps * N], far[:steps * N], profile=phi, reduction_db=20.0)
    stage = np.concatenate([np.zeros(DO.D, np.float32), stage])[:steps * N]
    ref_in = engine.agc(stage, FS)
    b = made.create()
    out_a = _push(engine, a, _chunks(mic)[:steps], before=lambda k: engine.session_echo_reference(a, _chunks(far)[k]))
    out_b = _push(engine, b, _chunks(ref_in)[:steps])
    assert float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert _same(out_a, out_b)


def test_submit_collect_and_push_device_are_the_push_path(engine, made):
    import torch
    steps = 12
    x = _speech((steps + 1) * T, stream=1021)
    chunks = _chunks(x)[:steps]
    want = _push(engine, made.create(), _chunks(engine.agc(x[:steps * N], FS)))
    a = _agc_session(engine, made)
    buf = np.empty(engine.session_io_geometry(a)['max_out'])
    tickets, got = [], []
    for c in chunks:                                    # up to five chunks in flight
        tickets.append(engine.session_submit(a, c))
        if len(tickets) == 5:
            got += [engine.session_collect(a, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(a, t, buf).copy() for t in tickets]
    assert _same(got, want)
    b = _agc_session(engine, made)
    cap = engine.session_io_geometry(b)['max_out']
    d_in = torch.from_numpy(np.stack(chunks)).cuda()
    d_out = torch.zeros((steps, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((steps, 1), dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    for k in range(steps):
        engine.session_push_device(b, d_in[k].data_ptr(), N, d_out[k].data_ptr(), cap, d_n[k].data_ptr())
    engine.synchronize()
    n = d_n.cpu().numpy().ravel()
    out = d_out.cpu().numpy()
    assert _same([out[k, :n[k]] for k in range(steps)], want)


# ---- 3 and 5 ------------------------------------------------------------------------------------------------------------------
def test_a_setting_change_lands_on_the_next_submitted_step_and_the_meter_is_the_oracles(engine, made):
    steps, j1 = 10, 4
    x = _speech((steps + 1) * T, stream=1031)
    chunks = _chunks(x)[:steps]
    s0, s1 = (-26.0, 20.0, -50.0), (-14.0, 8.0, -45.0)
    piped = _agc_session(engine, made, s0)
    tickets, got = [], []
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    for k, c in enumerate(chunks):                     # chunks in flight: five submitted before the first collect
        if k == j1:
            engine.session_set_agc(piped, *s1)
            assert engine.session_get_agc(piped)['target_db'] == -14.0
        tickets.append(engine.session_submit(piped, c))
        if k == 4:
            got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
    # block m uses the settings of the step that brings its last sample
    nb = steps * N // A.B
    late = ((np.arange(nb) + 1) * A.B - 1) // N >= j1
    cols = [np.where(late, v1, v0) for v0, v1 in zip(s0, s1)]
    ref_in = A.agc(x[:steps * N], FS, *cols)
    assert not np.array_equal(ref_in, A.agc(x[:steps * N], FS, *s0))
    assert _same(got, _push(engine, made.create(), _chunks(ref_in)))
    # the meter after each blocking step is the streaming oracle's
    blocking = _agc_session(engine, made, s0)
    st = A.AgcStream(FS, *s0)
    for k, c in enumerate(chunks):
        if k == j1:
            engine.session_set_agc(blocking, *s1)
            st.set(*s1)
        engine.session_push(blocking, c)
        st.push(c)
        level, gain, active = engine.session_agc_stats(blocking)
        want = st.last_meter
        assert active == want[2] and math.isclose(level, want[0], rel_tol=1e-14) and math.isclose(gain, want[1], rel_tol=1e-14, abs_tol=1e-14), k
    print(f'meter after {steps} steps: level {level:.2f} dB, gain {gain:+.2f} dB, {active} active blocks')


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
def test_group_members_and_voice_switches_keep_the_agc(engine, made, full_models, second_voice_files):
    steps, switch_at = 8, 4
    x = _speech((steps + 1) * T, stream=1041)
    chunks = _chunks(x)[:steps]
    engine.set_precision('fp32')
    alone = _push(engine, _agc_session(engine, made), chunks)
    a, b = _agc_session(engine, made), _agc_session(engine, made, (-20.0, 10.0, -60.0))
    gid = engine.group_create([a, b])
    made.gids.append(gid)
    bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(2)]
    got = []
    for k in range(steps):
        outs = engine.group_collect(gid, engine.group_submit(gid, [chunks[k], chunks[-1 - k]]), bufs)
        got.append(outs[0].copy())
    assert _same(got, alone)
    engine.set_precision('fp16')
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    reference = made.create(voice=v1)
    want = _push(engine, reference, _chunks(engine.agc(x[:steps * N], FS)),
                 before=lambda k: k == switch_at and engine.session_set_voice(reference, v2))
    switched = _agc_session(engine, made, voice=v1)
    out = _push(engine, switched, chunks, before=lambda k: k == switch_at and engine.session_set_voice(switched, v2))
    assert _same(out, want)


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def _launch_windows(out_dir):
    """Child process of the launch-count test: returns (kernels the profiler saw, change of engine.launch_count) over 12 steps of a
    plain session fed the whole-signal output (the same kernels downstream), of a session with the AGC fed the input, and of a plain
    one after it."""
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    _load(engine, synthetic.write_synthetic_models(out_dir / 'models', seed=0))
    engine.set_precision('fp16')
    steps = 12
    x = _speech((steps + 1) * T, stream=1051)
    controlled = _chunks(engine.agc(x[:steps * N], FS))
    counts = {}
    for name, chunks in (('plain', controlled), ('agc', _chunks(x)[:steps]), ('plain_after', controlled)):
        sid = engine.session_create(_cfg())
        if name == 'agc':
            engine.session_agc(sid)
        counts[name] = _window(engine, out_dir, lambda: _push(engine, sid, chunks))
        engine.session_destroy(sid)
    return counts


def test_one_kernel_per_step_and_none_for_other_sessions(tmp_path):
    counts = _run_child(tmp_path, 'test_gpu_agc', '_launch_windows')
    for name, (seen, counted) in counts.items():
        print(f'{name}: {counted} kernels counted over 12 steps, {seen} seen by the profiler')
        assert seen == counted, name
    assert counts['agc'][1] - counts['plain'][1] == 1 * 12
    assert counts['plain_after'][1] == counts['plain'][1]


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 5
    x = _speech((steps + 1) * T, stream=1061)
    chunks = _chunks(x)[:steps]
    sid, twin, plain = _agc_session(engine, made), _agc_session(engine, made), made.create()

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    fresh = made.create()
    bad = [(-5.0, 20.0, -50.0), (-41.0, 20.0, -50.0), (math.nan, 20.0, -50.0), (-26.0, -0.5, -50.0), (-26.0, 30.5, -50.0),
           (-26.0, math.inf, -50.0), (-26.0, 20.0, -19.0), (-26.0, 20.0, -81.0), (-26.0, 20.0, math.nan)]
    for s in bad:
        refused(lambda: engine.session_agc(fresh, *s))
        refused(lambda: engine.agc(x[:1000], FS, *s))
    refused(lambda: engine.agc(x[:1000], 0))
    for call in (lambda: engine.session_set_agc(plain, -20.0, 10.0, -50.0), lambda: engine.session_get_agc(plain),
                 lambda: engine.session_agc_stats(plain), lambda: engine.session_agc(99999), lambda: engine.session_get_agc(99999)):
        refused(call)
    outs = _push(engine, sid, chunks[:2])
    refused(lambda: engine.session_agc(sid))                  # ran a step
    refused(lambda: engine.session_agc(twin))                 # enabled twice
    before = engine.session_get_agc(sid)
    for s in bad:
        refused(lambda: engine.session_set_agc(sid, *s))
    assert engine.session_get_agc(sid) == before
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_agc(s)
        engine.session_set_input_rate(s, 48000)
        engine.session_push(s, np.zeros(engine.session_io_geometry(s)['n_in'], np.float32))
        engine.session_push(s, np.zeros(engine.session_io_geometry(s)['n_in'], np.float32))
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with the AGC')
    assert abs(grown) < 4.0


# ---- 8 ------------------------------------------------------------------------------------------------------------------------
def test_run_agc_is_the_pipelines_agc(engine, small_models, tmp_path):
    import yaml
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config
    from realtime_yukarin_b200.converter import YukarinConverter
    from realtime_yukarin_b200.worker import RealtimePipeline
    _load(engine, small_models)
    engine.set_precision('fp16')
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=0.5, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], extract_f0_mode='world')
    paths = {k: str(small_models[k]) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                               'stage1_config_path', 'stage2_model_path', 'stage2_config_path')}
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(dict(fields, **paths)))
    wave_io.write_wav(tmp_path / 'quiet.wav', _golden(4.0, db=-20.0), FS)
    run_mod.main(['--config_path', str(tmp_path / 'config.yaml'), '--wav_in', str(tmp_path / 'quiet.wav'), '--wav_out',
                  str(tmp_path / 'agc.wav'), '--agc', '-22', '--agc_max_gain', '15'])
    config = Config.from_yaml(tmp_path / 'config.yaml')
    param = YukarinConverter.make_yukarin_converter(**paths).acoustic_converter.config.dataset.acoustic_param
    wave = wave_io.load_wave(tmp_path / 'quiet.wav', config.input_rate, engine=engine).wave

    def pipeline_run(**kw):
        pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, **kw)
        got = []
        try:
            for i in range(len(wave) // config.in_audio_chunk):
                got.append(pipe.process(wave[i * config.in_audio_chunk:(i + 1) * config.in_audio_chunk]))
            got.extend(pipe.drain())
            pipe.flush()
            stats = pipe.agc_stats() if kw else None
        finally:
            pipe.close()
        return np.concatenate(got), stats

    def played(w):
        """the output chunks that carry sound: where the loop plays silence because nothing was ready yet depends on timing"""
        w = np.asarray(w)
        frames = w[:len(w) // config.out_audio_chunk * config.out_audio_chunk].reshape(-1, config.out_audio_chunk)
        return frames[np.any(frames != 0, axis=1)]

    mine, stats = pipeline_run(agc=-22.0, agc_max_gain_db=15.0)
    plain, _ = pipeline_run()
    ran = wave_io.load_wave(tmp_path / 'agc.wav', FS, engine=engine).wave
    assert len(played(mine)) >= 10 and np.array_equal(played(ran), played(mine))
    assert not np.array_equal(played(plain), played(mine))
    print(f'run.py --agc -22 --agc_max_gain 15 on speech at -20 dB (input_scale 0.5): level {stats[0]:.2f} dB, gain {stats[1]:+.2f} dB')
    assert stats[1] > 5.0
