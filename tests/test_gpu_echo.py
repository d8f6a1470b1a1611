"""Echo cancellation of a streaming session (ryk_session_echo_cancel and its calls) and the whole-signal ryk_echo_cancel, at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models.

  * ryk_echo_cancel is the FP64 oracle (tests/echo_oracle.py) to FP32 output rounding, bins whose error stands out are reported;
  * a session with the canceller is bitwise a session without it fed concat(zeros(511), ryk_echo_cancel(mic, far)), at a 24 kHz and
    a 48 kHz device input rate, with and without noise suppression, in both enabling orders;
  * a suppression change lands on the next submitted step; a group member is bitwise the session alone; a voice switch keeps the
    filter's state;
  * four kernels per step (five with noise suppression) and none for other sessions; refusals change nothing; cycles return memory;
  * a closed loop through run.audio_loop converges, and run.py --echo_cancel is RealtimePipeline(echo_cancel=True).
"""
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import RykError

from . import denoise_oracle as DO
from . import echo_oracle as E
from .test_gpu_f0_control import (EXTRA, FS, N, T, _cfg, _new_voice, _push, _same, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_launch_count import _run_child, _window
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'


def _far(seconds):
    x, rate = wave_io.read_wav(GOLDEN)
    assert rate == FS
    x = np.tile(np.asarray(x, np.float32), int(np.ceil(seconds * FS / len(x)) + 1))[:round(seconds * FS)]
    return x


def _scene(seconds, stream, delay_ms=30, near_db=-6.0, talk_from=1.0):
    """(mic, far) float32 at 24 kHz: the far end through a synthetic room, plus near-end speech from `talk_from` s at near_db under the
    echo"""
    far = _far(seconds)
    echo = E.echo_of(far, E.room_ir(delay_ms, seed=stream))
    near = synthetic.synthetic_speech(seconds, stream=stream)
    near = near / np.sqrt(np.mean(near ** 2)) * np.sqrt(np.mean(echo ** 2)) * 10 ** (near_db / 20)
    t0 = round(talk_from * FS)
    mic = echo.copy()
    mic[t0:] += near[:len(mic) - t0]
    return mic.astype(np.float32), far


def _chunks(x, n=N):
    return [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(len(x) // n)]


def _cancelled_input(engine, mic, far, phi=None, delay=DO.D, **kw):
    """what a session with the canceller analyses: concat(zeros(delay), ryk_echo_cancel(mic, far)), as long as mic"""
    z = engine.echo_cancel(mic, far, profile=phi, **kw)
    return np.concatenate([np.zeros(delay, np.float32), z])[:len(mic)]


def _push_echo(engine, sid, chunks, fars, before=None):
    """blocking pushes with the far end of each chunk handed in first"""
    def ref(k):
        if before:
            before(k)
        engine.session_echo_reference(sid, fars[k])
    return _push(engine, sid, chunks, before=ref)


def _cancelling(engine, made, taps=32, phi=None, voice=0):
    sid = made.create(voice=voice)
    engine.session_echo_cancel(sid, taps=taps)
    if phi is not None:
        engine.session_denoise(sid)
        engine.session_set_noise_profile(sid, phi)
    return sid


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_the_whole_signal_call_is_the_oracle(engine):
    mic, far = _scene(3.0, stream=801)
    phi = DO.frame_powers(mic, 3, 60).mean(axis=0)
    worst = 0.0
    for kw in (dict(taps=32), dict(taps=16, delay_frames=5, suppression_db=15.0), dict(taps=64, phi=phi, reduction_db=20.0),
               dict(taps=1)):
        got = engine.echo_cancel(mic, far, **{('profile' if k == 'phi' else k): v for k, v in kw.items()})
        want = E.echo_cancel(mic, far, **kw)
        diff = got.astype(np.float64) - want.astype(np.float64)
        err = float(np.max(np.abs(diff)))
        # bins whose error stands out: where a copy decision of the two-path control went the other way on the device
        P = DO.frame_powers(diff, 0, len(diff) // DO.H).sum(axis=0)
        flipped = np.nonzero(P > 1e-3 * max(P.sum(), 1e-300))[0] if err > 1e-6 else []
        print(f'{kw.get("taps")} taps, delay {kw.get("delay_frames", 0)}, suppression {kw.get("suppression_db", 0.0)} dB, '
              f'noise profile {"phi" in kw}: max abs difference {err:.2e}; bins standing out: {list(flipped)}')
        assert err <= 2e-5, (kw, err, list(flipped))
        worst = max(worst, err)
    print(f'ryk_echo_cancel vs the FP64 oracle: max abs difference {worst:.2e}')
    assert np.array_equal(engine.echo_cancel(mic, far), engine.echo_cancel(mic, far))
    # it cancels: the far end alone leaves a residual far under the echo after the first second
    echo = E.echo_of(far, E.room_ir(30, seed=801)).astype(np.float32)
    z = engine.echo_cancel(echo, far)
    assert -E.level_db(z[2 * FS:], echo[2 * FS:]) > 20.0


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rate, denoise, order', [(FS, False, 'echo'), (FS, True, 'echo'), (FS, True, 'denoise'), (48000, False, 'rate'),
                                                  (48000, True, 'echo')])
def test_the_stream_is_the_whole_signal_bitwise(engine, made, rate, denoise, order):
    steps = 20
    mic24, far24 = _scene((steps + 1) * T, stream=811)
    phi = DO.frame_powers(mic24, 3, 60).mean(axis=0) if denoise else None
    a = made.create()
    calls = dict(echo=lambda: engine.session_echo_cancel(a, taps=32), denoise=lambda: engine.session_denoise(a),
                 rate=lambda: engine.session_set_input_rate(a, rate))
    sequence = [order] + [c for c in ('echo', 'denoise', 'rate') if c != order]
    for c in sequence:
        if c == 'denoise' and not denoise or c == 'rate' and rate == FS:
            continue
        calls[c]()
    if denoise:
        engine.session_set_noise_profile(a, phi)
    geo = engine.session_io_geometry(a)
    if rate == FS:
        mic, far, model_mic, model_far = mic24, far24, mic24, far24
        assert geo['delay_in'] == DO.D
    else:
        mic, far = wave_io.resample(mic24, FS, rate, engine), wave_io.resample(far24, FS, rate, engine)
        d_rs = geo['delay_in'] - DO.D
        assert d_rs == wave_io.stream_input_geometry(rate, FS, T)[2]
        up, down = 1, 2
        taps = wave_io.resample_filter(up, down)
        model_mic, model_far = (np.concatenate([np.zeros(d_rs, np.float32), engine.resample_poly(s, up, down, taps)]) for s in (mic, far))
    b = made.create()
    ref_in = _cancelled_input(engine, model_mic[:steps * N], model_far[:steps * N], phi, reduction_db=20.0)
    out_a = _push_echo(engine, a, _chunks(mic, geo['n_in'])[:steps], _chunks(far, geo['n_in']))
    out_b = _push(engine, b, _chunks(ref_in)[:steps])
    assert sum(len(o) for o in out_a) > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert _same(out_a, out_b)
    frames, erle = engine.session_echo_stats(a)
    print(f'rate {rate}, denoise {denoise}, enabled {sequence}: last step {frames} frames, ERLE {erle:.1f} dB')
    assert frames == (steps * N) // DO.H - ((steps - 1) * N) // DO.H
    # and the canceller does something: the stream without it differs
    c = made.create()
    if rate != FS:
        engine.session_set_input_rate(c, rate)
    if denoise:
        engine.session_denoise(c)
        engine.session_set_noise_profile(c, phi)
    assert not _same(out_a, _push(engine, c, _chunks(mic, geo['n_in'])[:steps]))


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def test_a_suppression_change_lands_on_the_next_step(engine, made):
    steps, j1 = 8, 3
    mic, far = _scene((steps + 1) * T, stream=821)
    chunks, fars = _chunks(mic)[:steps], _chunks(far)
    piped, blocking, never = (_cancelling(engine, made) for _ in range(3))
    tickets, got = [], []
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    for k, c in enumerate(chunks):                     # chunks in flight: five submitted before the first collect
        if k == j1:
            engine.session_set_echo_suppression(piped, 25.0)
        engine.session_echo_reference(piped, fars[k])
        tickets.append(engine.session_submit(piped, c))
        if k == 4:
            got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
    out_blocking = _push_echo(engine, blocking, chunks, fars, before=lambda k: k == j1 and engine.session_set_echo_suppression(blocking, 25.0))
    out_never = _push_echo(engine, never, chunks, fars)
    assert _same(got, out_blocking)
    assert _same(got[:j1], out_never[:j1]) and not _same(got[j1:], out_never[j1:])
    # 0 dB is the linear canceller exactly: setting it back restores the plain stream's filter output from then on
    s0 = _cancelling(engine, made)
    engine.session_set_echo_suppression(s0, 0.0)
    assert _same(_push_echo(engine, s0, chunks, fars), out_never)


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
def test_group_members_and_voice_switches_keep_the_filter(engine, made, full_models, second_voice_files):
    steps, switch_at = 8, 4
    mic, far = _scene((steps + 1) * T, stream=831)
    chunks, fars = _chunks(mic)[:steps], _chunks(far)
    engine.set_precision('fp32')
    alone = _push_echo(engine, _cancelling(engine, made), chunks, fars)
    a, b = _cancelling(engine, made), made.create()
    gid = engine.group_create([a, b])
    made.gids.append(gid)
    bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(2)]
    got = []
    for k in range(steps):
        engine.session_echo_reference(a, fars[k])
        outs = engine.group_collect(gid, engine.group_submit(gid, [chunks[k], chunks[-1 - k]]), bufs)
        got.append(outs[0].copy())
    assert _same(got, alone)
    # a voice switch keeps the filter's state: bitwise a session without the canceller fed the whole-signal output, switched alike
    engine.set_precision('fp16')
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    switched = _cancelling(engine, made, voice=v1)
    reference = made.create(voice=v1)
    ref_in = _chunks(_cancelled_input(engine, mic[:steps * N], far[:steps * N]))
    out_s = _push_echo(engine, switched, chunks, fars, before=lambda k: k == switch_at and engine.session_set_voice(switched, v2))
    out_r = _push(engine, reference, ref_in, before=lambda k: k == switch_at and engine.session_set_voice(reference, v2))
    assert _same(out_s, out_r)


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def _launch_windows(out_dir):
    """Child process of the launch-count test: returns (kernels the profiler saw, change of engine.launch_count) over 12 steps of sessions
    without the canceller fed the whole-signal output (the same kernels downstream) and with it, with and without noise suppression."""
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    _load(engine, synthetic.write_synthetic_models(out_dir / 'models', seed=0))
    engine.set_precision('fp16')
    steps = 12
    mic, far = _scene((steps + 1) * T, stream=841)
    chunks, fars = _chunks(mic)[:steps], _chunks(far)
    phi = DO.frame_powers(mic, 3, 60).mean(axis=0)
    counts = {}
    # plain / plain_dn: no canceller, fed the whole-signal output without / with noise suppression
    for name in ('plain', 'echo', 'plain_dn', 'both'):
        sid = engine.session_create(_cfg())
        fed = chunks
        if name in ('echo', 'both'):
            engine.session_echo_cancel(sid)
        if name == 'both':
            engine.session_denoise(sid)
            engine.session_set_noise_profile(sid, phi)
        if name.startswith('plain'):
            fed = _chunks(_cancelled_input(engine, mic[:steps * N], far[:steps * N], phi if name == 'plain_dn' else None))
        if name in ('echo', 'both'):
            counts[name] = _window(engine, out_dir, lambda: _push_echo(engine, sid, fed, fars))
        else:
            counts[name] = _window(engine, out_dir, lambda: _push(engine, sid, fed))
        engine.session_destroy(sid)
    return counts


def test_four_kernels_per_step_and_none_for_other_sessions(tmp_path):
    counts = _run_child(tmp_path, 'test_gpu_echo', '_launch_windows')
    for name, (seen, counted) in counts.items():
        print(f'{name}: {counted} kernels counted over 12 steps, {seen} seen by the profiler')
        assert seen == counted, name
    assert counts['echo'][1] - counts['plain'][1] == 4 * 12
    assert counts['both'][1] - counts['plain_dn'][1] == 5 * 12


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 5
    mic, far = _scene((steps + 1) * T, stream=851)
    chunks, fars = _chunks(mic)[:steps], _chunks(far)
    sid, twin, plain = _cancelling(engine, made), _cancelling(engine, made), made.create()

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    fresh = made.create()
    for taps, delay in ((0, 0), (65, 0), (32, -1), (32, 257)):
        refused(lambda: engine.session_echo_cancel(fresh, taps=taps, delay_ms=delay * DO.H * 1000.0 / FS))
        refused(lambda: engine.echo_cancel(mic[:1000], far[:1000], taps=taps, delay_frames=delay))
    assert engine.session_io_geometry(fresh)['delay_in'] == 0
    outs = _push_echo(engine, sid, chunks[:2], fars)
    refused(lambda: engine.session_echo_cancel(sid))             # ran a step
    refused(lambda: engine.session_echo_cancel(99999))
    refused(lambda: engine.session_echo_reference(sid, fars[2][:-1]))
    refused(lambda: engine.session_echo_reference(sid, np.concatenate([fars[2], fars[2][:1]])))
    for db in (float('nan'), float('inf'), -0.5, 40.5):
        refused(lambda: engine.session_set_echo_suppression(sid, db))
        refused(lambda: engine.echo_cancel(mic[:1000], far[:1000], suppression_db=db))
    for call in (lambda: engine.session_echo_reference(plain, fars[0]), lambda: engine.session_set_echo_suppression(plain, 10.0),
                 lambda: engine.session_echo_stats(plain), lambda: engine.session_set_echo_suppression(99999, 10.0)):
        refused(call)
    twice = made.create()
    engine.session_echo_cancel(twice)
    refused(lambda: engine.session_echo_cancel(twice))
    assert engine.session_io_geometry(plain)['delay_in'] == 0
    outs += _push_echo(engine, sid, chunks[2:], fars[2:])
    assert _same(outs, _push_echo(engine, twin, chunks, fars))
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_echo_cancel(s, taps=64, delay_ms=200.0)
        engine.session_echo_reference(s, fars[0])
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with the canceller')
    assert abs(grown) < 4.0


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def _config_file(small_models, tmp_path):
    import yaml
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], extract_f0_mode='world')
    paths = {k: str(small_models[k]) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                               'stage1_config_path', 'stage2_model_path', 'stage2_config_path')}
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(dict(fields, **paths)))
    return tmp_path / 'config.yaml', paths


def test_closed_loop_converges_and_run_is_the_pipeline(engine, small_models, tmp_path, monkeypatch):
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config
    from realtime_yukarin_b200.converter import YukarinConverter
    from realtime_yukarin_b200.worker import RealtimePipeline
    _load(engine, small_models)
    engine.set_precision('fp16')
    # Which chunk's output is ready when process() looks depends on timing, and with echo cancellation the played stream is the far
    # end, so the runs compared here finish each chunk before taking its output
    process = RealtimePipeline.process
    monkeypatch.setattr(RealtimePipeline, 'process', lambda self, w, block=False: process(self, w, block=True))
    path, paths = _config_file(small_models, tmp_path)
    config = Config.from_yaml(path)
    param = YukarinConverter.make_yukarin_converter(**paths).acoustic_converter.config.dataset.acoustic_param
    n = config.in_audio_chunk
    steps, talk = 40, 15
    near = synthetic.synthetic_speech((steps + 1) * T, stream=861).astype(np.float32)
    near[talk * n:] = 0.0                              # the speaker stops after 4.5 s; the converted voice goes on playing
    ir = E.room_ir(30, seed=861)

    # closed loop: the microphone picks up the near-end voice and the room's echo of everything played so far
    pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, echo_cancel=True)
    played, erle = [np.zeros(n, np.float32)], []
    pos = [0]

    def read_chunk():
        k = pos[0]
        if k >= steps:
            return None
        pos[0] = k + 1
        stream = np.concatenate(played)
        echo = E.echo_of(stream, ir)[k * n:(k + 1) * n]
        return (near[k * n:(k + 1) * n] + echo).astype(np.float32)

    def write_chunk(w):
        played.append(np.asarray(w, np.float32))
        erle.append(pipe.echo_stats()[1])
    try:
        assert run_mod.audio_loop(pipe, read_chunk, write_chunk) == steps
    finally:
        pipe.close()
    loud = sum(1 for p in played if np.abs(p).max() > 1e-2)
    print(f'closed loop: {loud} of {steps} chunks played sound; ERLE per chunk (dB): {[round(e, 1) for e in erle]}')
    assert loud >= steps // 2
    # the same loop on the CPU oracle (tests/test_echo.py, 30 chunks) stays at -0.0 dB or above and ends at 19.5-20.8 dB
    assert min(erle) >= -1.0 and float(np.mean(erle[-10:])) >= 12.0

    # run.py --echo_cancel 16 --echo_delay 10 --echo_suppression 6 is RealtimePipeline with the same settings, bitwise
    wave_io.write_wav(tmp_path / 'near.wav', near, FS)
    run_mod.main(['--config_path', str(path), '--wav_in', str(tmp_path / 'near.wav'), '--wav_out', str(tmp_path / 'out.wav'),
                  '--echo_cancel', '16', '--echo_delay', '10', '--echo_suppression', '6'])
    wave = wave_io.load_wave(tmp_path / 'near.wav', config.input_rate, engine=engine).wave
    pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, echo_cancel=True, echo_taps=16, echo_delay_ms=10.0,
                            echo_suppression=6.0)
    mine = []
    try:
        for i in range(len(wave) // n):
            mine.append(pipe.process(wave[i * n:(i + 1) * n]))
        mine.extend(pipe.drain())
    finally:
        pipe.close()
    ran = wave_io.load_wave(tmp_path / 'out.wav', FS, engine=engine).wave
    mine = np.concatenate(mine)
    assert np.abs(mine).max() > 1e-2
    assert len(ran) == len(mine) and np.array_equal(ran, mine)
