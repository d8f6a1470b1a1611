"""The output limiter of a streaming session (ryk_session_limiter and its calls) and the whole-signal ryk_limit, at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models.

  * ryk_limit is the FP64 oracle (tests/limiter_oracle.py) bit for bit at 24 and 48 kHz over several look-aheads, holds and ceilings;
  * a limited session is bitwise concat(zeros(L), ryk_limit(y)) of the same session unlimited: at 24 kHz, at a 48 kHz output rate in
    both enabling orders, through push, submit / collect and push_device; below the ceiling it is the unlimited stream delayed by L;
  * a setting change made with chunks in flight lands on the next submitted step; group members are the sessions alone; a voice switch
    keeps the limiter's state; the meter is the oracle's;
  * three kernels per step and none for other sessions; refusals change nothing; cycles return memory;
  * RealtimePipeline through run.audio_loop with a large output_scale plays nothing above the ceiling, and does without the limiter.
"""
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import RykError

from . import limiter_oracle as LO
from .test_gpu_f0_control import (EXTRA, FS, N, T, _cfg, _new_voice, _push, _same, _speech, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_launch_count import _run_child, _window
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

LA, HOLD = 5.0, 50.0


def _flat(outs):
    return np.concatenate(outs) if outs else np.zeros(0)


def _limited(engine, made, rate=FS, order='limiter', la=LA, hold=HOLD, voice=0):
    sid = made.create(voice=voice)
    if rate != FS and order == 'rate':
        engine.session_set_output_rate(sid, rate)
    engine.session_limiter(sid, lookahead_ms=la, hold_ms=hold)
    if rate != FS and order != 'rate':
        engine.session_set_output_rate(sid, rate)
    return sid


def _plain(engine, made, rate=FS, voice=0):
    sid = made.create(voice=voice)
    if rate != FS:
        engine.session_set_output_rate(sid, rate)
    return sid


def _engaging_gain(y, ceiling_db=-1.0, over=4.0):
    """a gain under which the loudest sample of y plays `over` times the ceiling"""
    return over * LO.ceiling(ceiling_db) / float(np.max(np.abs(y)))


def _expected(engine, y, rate, gain, ceiling_db=-1.0, la=LA, hold=HOLD):
    L, _ = LO.shape(rate, la, hold)
    return np.concatenate([np.zeros(L), engine.limit(y, rate, la, hold, ceiling_db, gain)])[:len(y)]


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_the_whole_signal_call_is_the_oracle(engine):
    x, fs = wave_io.read_wav(Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav')
    speech = 4.0 * np.asarray(x, np.float64)
    rng = np.random.default_rng(7)
    imp = rng.normal(0, 0.05, 50000)
    imp[rng.integers(0, 50000, 60)] = rng.uniform(-5, 5, 60)
    cases = 0
    for rate in (24000, 48000):
        for la, hold in ((5.0, 50.0), (0.5, 0.0), (10.0, 500.0), (2.5, 7.0), (1.0, 1000 / rate)):
            for db, gain in ((-1.0, 1.0), (-12.0, 2.5), (0.0, 0.3), (-24.0, 1.0)):
                for y in (speech, imp):
                    got = engine.limit(y, rate, la, hold, db, gain)
                    want = LO.limit(y, rate, la, hold, db, gain)
                    assert np.array_equal(got, want), (rate, la, hold, db, gain, float(np.max(np.abs(got - want))))
                    assert np.all(np.abs(gain * got) <= LO.ceiling(db) * (1 + 1e-12))
                    cases += 1
    print(f'ryk_limit is the FP64 oracle bit for bit in {cases} cases')


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rate, order', [(FS, 'limiter'), (48000, 'limiter'), (48000, 'rate')])
def test_the_stream_is_the_whole_signal_bitwise(engine, made, rate, order):
    steps = 16
    chunks = _speech(steps, stream=901)
    y = _push(engine, _plain(engine, made, rate), chunks)
    yf = _flat(y)
    gain = _engaging_gain(yf)
    a = _limited(engine, made, rate, order)
    engine.session_set_limiter(a, -1.0, gain)
    got = engine.session_get_limiter(a)
    L, R = LO.shape(rate, LA, HOLD)
    assert got == dict(ceiling_db=-1.0, gain=gain, lookahead=L, hold=R)
    assert engine.session_io_geometry(a)['max_out'] == engine.session_io_geometry(made.sids[-2])['max_out']
    outs, stats = [], []
    buf = np.empty(engine.session_io_geometry(a)['max_out'])
    for c in chunks:
        outs.append(engine.session_push(a, c, buf).copy())
        stats.append(engine.session_limiter_stats(a))
    assert [len(o) for o in outs] == [len(o) for o in y]
    want = _expected(engine, yf, rate, gain)
    assert np.array_equal(_flat(outs), want)
    assert not np.array_equal(want, np.concatenate([np.zeros(L), yf])[:len(yf)]), 'the limiter never engaged'
    assert np.all(np.abs(gain * _flat(outs)) <= LO.ceiling(-1.0) * (1 + 1e-12))
    # the meter of each step is the oracle's over the samples it returned
    _, g = LO.limit(yf, rate, LA, HOLD, -1.0, gain, return_gain=True)
    a0 = 0
    for o, (red, lim) in zip(outs, stats):
        t = np.arange(a0, a0 + len(o)) - L
        want_red, want_lim = LO.meter(g[t[t >= 0]])
        assert lim == want_lim and np.isclose(red, want_red, rtol=1e-12, atol=0)
        a0 += len(o)
    assert sum(s[1] for s in stats) > 0
    print(f'rate {rate}: L {L}, R {R}, gain {gain:.3f}; reductions per step (dB): {[round(s[0], 2) for s in stats]}')


def test_submit_collect_and_push_device_are_the_push_path(engine, made):
    import torch
    steps = 12
    chunks = _speech(steps, stream=911)
    y = _flat(_push(engine, _plain(engine, made), chunks))
    gain = _engaging_gain(y)
    want = _expected(engine, y, FS, gain)
    # submit / collect with up to five chunks in flight
    a = _limited(engine, made)
    engine.session_set_limiter(a, -1.0, gain)
    buf = np.empty(engine.session_io_geometry(a)['max_out'])
    tickets, got = [], []
    for k, c in enumerate(chunks):
        tickets.append(engine.session_submit(a, c))
        if len(tickets) == 5:
            got += [engine.session_collect(a, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(a, t, buf).copy() for t in tickets]
    assert np.array_equal(_flat(got), want)
    # device-resident pushes
    b = _limited(engine, made)
    engine.session_set_limiter(b, -1.0, gain)
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
    assert np.array_equal(np.concatenate([out[k, :n[k]] for k in range(steps)]), want)


def test_below_the_ceiling_the_stream_is_the_plain_one_delayed(engine, made):
    steps = 10
    chunks = _speech(steps, stream=921)
    y = _flat(_push(engine, _plain(engine, made), chunks))
    gain = 0.5 * LO.ceiling(-1.0) / float(np.max(np.abs(y)))
    a = _limited(engine, made, hold=500.0)
    engine.session_set_limiter(a, -1.0, gain)
    out = _flat(_push(engine, a, chunks))
    L, _ = LO.shape(FS, LA, 500.0)
    assert np.array_equal(out, np.concatenate([np.zeros(L), y])[:len(y)])
    assert engine.session_limiter_stats(a) == (0.0, 0)


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def test_a_setting_change_lands_on_the_next_submitted_step(engine, made):
    steps, j1 = 9, 3
    chunks = _speech(steps, stream=931)
    y_steps = _push(engine, _plain(engine, made), chunks)
    y = _flat(y_steps)
    g1, g2 = _engaging_gain(y, over=2.0), _engaging_gain(y, over=6.0)
    piped = _limited(engine, made)
    engine.session_set_limiter(piped, -1.0, g1)
    tickets, got = [], []
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    for k, c in enumerate(chunks):                     # chunks in flight: five submitted before the first collect
        if k == j1:
            engine.session_set_limiter(piped, -6.0, g2)
            assert engine.session_get_limiter(piped)['ceiling_db'] == -6.0
        tickets.append(engine.session_submit(piped, c))
        if k == 4:
            got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
    # the oracle with per-sample settings: g0 of the samples step k returned from upstream uses step k's settings
    n_before = sum(len(o) for o in y_steps[:j1])
    cdb = np.where(np.arange(len(y)) < n_before, -1.0, -6.0)
    gains = np.where(np.arange(len(y)) < n_before, g1, g2)
    L, _ = LO.shape(FS, LA, HOLD)
    want = np.concatenate([np.zeros(L), LO.limit(y, FS, LA, HOLD, cdb, gains)])[:len(y)]
    assert np.array_equal(_flat(got), want)
    blocking = _limited(engine, made)
    engine.session_set_limiter(blocking, -1.0, g1)
    out_b = _push(engine, blocking, chunks, before=lambda k: k == j1 and engine.session_set_limiter(blocking, -6.0, g2))
    assert _same(got, out_b)


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
def test_group_members_and_voice_switches_keep_the_limiter(engine, made, full_models, second_voice_files):
    steps, switch_at = 8, 4
    chunks = _speech(steps, stream=941)
    engine.set_precision('fp32')
    y = _flat(_push(engine, _plain(engine, made), chunks))
    gain = _engaging_gain(y)
    alone_sid = _limited(engine, made)
    engine.session_set_limiter(alone_sid, -1.0, gain)
    alone = _push(engine, alone_sid, chunks)
    a, b = _limited(engine, made), _limited(engine, made)
    engine.session_set_limiter(a, -1.0, gain)
    engine.session_set_limiter(b, -3.0, gain)
    gid = engine.group_create([a, b])
    made.gids.append(gid)
    bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(2)]
    got = []
    for k in range(steps):
        outs = engine.group_collect(gid, engine.group_submit(gid, [chunks[k], chunks[-1 - k]]), bufs)
        got.append(outs[0].copy())
    assert _same(got, alone)
    # a voice switch keeps the limiter's state: bitwise the whole-signal limiter of an unlimited session switched alike
    engine.set_precision('fp16')
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    reference = _plain(engine, made, voice=v1)
    y_sw = _flat(_push(engine, reference, chunks, before=lambda k: k == switch_at and engine.session_set_voice(reference, v2)))
    gain = _engaging_gain(y_sw)
    switched = _limited(engine, made, voice=v1)
    engine.session_set_limiter(switched, -1.0, gain)
    out_s = _flat(_push(engine, switched, chunks, before=lambda k: k == switch_at and engine.session_set_voice(switched, v2)))
    assert np.array_equal(out_s, _expected(engine, y_sw, FS, gain))


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def _launch_windows(out_dir):
    """Child process of the launch-count test: returns (kernels the profiler saw, change of engine.launch_count) over 12 steps of a plain
    session, a limited one, and a plain one after the limited one ran on the same engine."""
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    _load(engine, synthetic.write_synthetic_models(out_dir / 'models', seed=0))
    engine.set_precision('fp16')
    steps = 12
    chunks = _speech(steps, stream=951)
    counts = {}
    for name in ('plain', 'limited', 'limited_48k', 'plain_48k', 'plain_after'):
        sid = engine.session_create(_cfg())
        if name.endswith('48k'):
            engine.session_set_output_rate(sid, 48000)
        if name.startswith('limited'):
            engine.session_limiter(sid, LA, HOLD)
            engine.session_set_limiter(sid, -1.0, 50.0)
        counts[name] = _window(engine, out_dir, lambda: _push(engine, sid, chunks))
        engine.session_destroy(sid)
    return counts


def test_three_kernels_per_step_and_none_for_other_sessions(tmp_path):
    counts = _run_child(tmp_path, 'test_gpu_limiter', '_launch_windows')
    for name, (seen, counted) in counts.items():
        print(f'{name}: {counted} kernels counted over 12 steps, {seen} seen by the profiler')
        assert seen == counted, name
    assert counts['limited'][1] - counts['plain'][1] == 3 * 12
    assert counts['limited_48k'][1] - counts['plain_48k'][1] == 3 * 12
    assert counts['plain_after'][1] == counts['plain'][1]


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 5
    chunks = _speech(steps, stream=961)
    sid, twin, plain = _limited(engine, made), _limited(engine, made), made.create()
    for s in (sid, twin):
        engine.session_set_limiter(s, -2.0, 30.0)

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    fresh = made.create()
    y = np.linspace(-3, 3, 5000)
    for la, hold in ((0.4, 50.0), (10.5, 50.0), (float('nan'), 50.0), (5.0, -1.0), (5.0, 500.5), (5.0, float('inf'))):
        refused(lambda: engine.session_limiter(fresh, la, hold))
        refused(lambda: engine.limit(y, FS, la, hold))
    refused(lambda: engine.limit(y, 0, LA, HOLD))
    for call in (lambda: engine.session_set_limiter(fresh, -1.0, 1.0), lambda: engine.session_get_limiter(fresh),
                 lambda: engine.session_limiter_stats(fresh), lambda: engine.session_limiter(99999), lambda: engine.session_get_limiter(99999)):
        refused(call)
    outs = _push(engine, sid, chunks[:2])
    refused(lambda: engine.session_limiter(sid))             # ran a step
    before = engine.session_get_limiter(sid)
    for db, gain in ((0.5, 1.0), (-24.5, 1.0), (float('nan'), 1.0), (-1.0, 0.0), (-1.0, -2.0), (-1.0, float('inf')), (-1.0, float('nan'))):
        refused(lambda: engine.session_set_limiter(sid, db, gain))
        refused(lambda: engine.limit(y, FS, LA, HOLD, db, gain))
    assert engine.session_get_limiter(sid) == before
    twice = made.create()
    engine.session_limiter(twice)
    refused(lambda: engine.session_limiter(twice))
    assert engine.session_get_limiter(twice)['ceiling_db'] == -1.0 and engine.session_get_limiter(twice)['gain'] == 1.0
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_limiter(s, 10.0, 500.0)
        engine.session_set_output_rate(s, 48000)
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with the limiter')
    assert abs(grown) < 4.0


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def _config_file(small_models, tmp_path, output_scale):
    import yaml
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=output_scale, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2],
                  extract_f0_mode='world')
    paths = {k: str(small_models[k]) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                               'stage1_config_path', 'stage2_model_path', 'stage2_config_path')}
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(dict(fields, **paths)))
    return tmp_path / 'config.yaml', paths


def test_the_pipeline_plays_under_the_ceiling_only_with_the_limiter(engine, small_models, tmp_path):
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config
    from realtime_yukarin_b200.converter import YukarinConverter
    from realtime_yukarin_b200.worker import RealtimePipeline
    _load(engine, small_models)
    engine.set_precision('fp16')
    path, paths = _config_file(small_models, tmp_path, output_scale=40.0)
    config = Config.from_yaml(path)
    param = YukarinConverter.make_yukarin_converter(**paths).acoustic_converter.config.dataset.acoustic_param
    n, steps = config.in_audio_chunk, 20
    x = synthetic.synthetic_speech((steps + 1) * T, stream=971).astype(np.float32)
    c = LO.ceiling(-1.0)

    def play(**kw):
        pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, **kw)
        played, pos, stats = [], [0], []

        def read_chunk():
            k = pos[0]
            if k >= steps:
                return None
            pos[0] = k + 1
            return x[k * n:(k + 1) * n]

        def write_chunk(w):
            played.append(np.asarray(w, np.float32))
            if kw:
                stats.append(pipe.limiter_stats())
        try:
            assert run_mod.audio_loop(pipe, read_chunk, write_chunk) == steps
            played += pipe.drain()
        finally:
            pipe.close()
        return np.concatenate(played), stats
    plain, _ = play()
    limited, stats = play(limiter=-1.0)
    print(f'output_scale 40: peak {np.max(np.abs(plain)):.2f} without the limiter, {np.max(np.abs(limited)):.4f} with it '
          f'(ceiling {c:.4f}); reductions per chunk (dB): {[round(s[0], 1) for s in stats]}')
    assert np.max(np.abs(plain)) > c
    assert np.max(np.abs(limited)) <= c * (1 + 2 ** -23)          # the float32 cast of the played chunk: half an ulp
    assert max(s[0] for s in stats) > 0.0
