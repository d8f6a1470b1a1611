"""Input noise suppression of a streaming session (ryk_session_denoise and its setters) and the whole-signal ryk_denoise, at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models.

  * ryk_denoise is the FP64 oracle (tests/denoise_oracle.py) to FP32 rounding, and the identity at reduction 0;
  * a session with the filter is bitwise a session without it fed concat(zeros(511), ryk_denoise(x)), at 24 and 48 kHz input;
  * learning: the profile is the oracle's mean over the same frames, bit-identical across runs and beside other work, counted down step
    by step, and applied from the step after the last learned frame exactly;
  * settings land on the step submitted after them; the stream is the oracle's filtered stream through StreamOracle;
  * the filter's state carries over group membership changes and voice switches;
  * three kernels per filtering step and none for other sessions; refusals change nothing; cycles return memory; run.py's flags.
"""
from pathlib import Path

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import RykError

from . import denoise_oracle as O
from .test_gpu_f0_control import (CFG, EXTRA, FS, N, TOL, T, _cfg, _new_voice, _push, _same, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_headline_parity import _rmse
from .test_gpu_launch_count import _run_child, _window
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu


def _noisy(seconds, stream, snr_db=10.0, lead=0.5):
    """synthetic speech after `lead` s of seeded white noise alone, the noise continuing under it at snr_db (float32)"""
    x = synthetic.synthetic_speech(seconds, stream=stream).astype(np.float64)
    n_lead = round(lead * FS)
    x = np.concatenate([np.zeros(n_lead), x[:len(x) - n_lead]])
    nz = np.random.default_rng(stream).standard_normal(len(x))
    scale = np.sqrt(np.mean(x[n_lead:] ** 2) / np.mean(nz ** 2) / 10 ** (snr_db / 10))
    return (x + scale * nz).astype(np.float32)


def _chunks(x, n=N):
    return [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(len(x) // n)]


def _profile(x, first=3, count=80):
    return O.frame_powers(x, first, count).mean(axis=0)


def _filtered_input(engine, x, reduction, phi, delay=O.D):
    """what a session with the filter analyses: concat(zeros(delay), ryk_denoise(x)), as long as x"""
    z = engine.denoise(x, reduction, phi)
    return np.concatenate([np.zeros(delay, np.float32), z])[:len(x)]


def _denoising(engine, made, reduction=20.0, phi=None, voice=0):
    sid = made.create(voice=voice)
    engine.session_denoise(sid)
    engine.session_set_denoise(sid, reduction)
    if phi is not None:
        engine.session_set_noise_profile(sid, phi)
    return sid


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_the_whole_signal_call_is_the_oracle(engine):
    x = _noisy(1.5, stream=701)
    phi = _profile(x)
    worst = 0.0
    for reduction in (0.0, 20.0, 40.0):
        for profile in (phi, None):
            got = engine.denoise(x, reduction, profile)
            want = O.denoise(x, reduction, profile)
            err = float(np.max(np.abs(got.astype(np.float64) - want.astype(np.float64))))
            assert err <= 1e-6, (reduction, profile is None, err)
            worst = max(worst, err)
            if reduction == 0.0 or profile is None:
                # the identity to rounding: within one FP32 ulp of x
                assert np.all(np.abs(got - x) <= np.spacing(np.abs(x))), reduction
            else:
                assert _rmse(got, x) > 1e-3
    print(f'ryk_denoise vs the FP64 oracle: max abs difference {worst:.2e} over the six cases')
    # the same call twice is bitwise the same
    assert np.array_equal(engine.denoise(x, 20.0, phi), engine.denoise(x, 20.0, phi))


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision, rate', [('fp32', FS), ('fp16', FS), ('fp16', 48000)])
def test_the_stream_is_the_whole_signal_bitwise(engine, made, precision, rate):
    steps = 32
    engine.set_precision(precision)
    x24 = _noisy((steps + 1) * T, stream=711)
    phi = _profile(x24)
    a = made.create()
    engine.session_denoise(a)
    if rate != FS:
        engine.session_set_input_rate(a, rate)         # after enabling: either order works
    engine.session_set_noise_profile(a, phi)
    geo = engine.session_io_geometry(a)
    if rate == FS:
        x, model = x24, x24
        assert geo['delay_in'] == O.D
    else:
        x = wave_io.resample(x24, FS, rate, engine)
        d_rs = geo['delay_in'] - O.D
        assert d_rs == wave_io.stream_input_geometry(rate, FS, T)[2]
        up, down = 1, 2
        model = np.concatenate([np.zeros(d_rs, np.float32), engine.resample_poly(x, up, down, wave_io.resample_filter(up, down))])
    b = made.create()
    ref_in = _filtered_input(engine, model[:steps * N], 20.0, phi)
    out_a = _push(engine, a, _chunks(x, geo['n_in'])[:steps])
    out_b = _push(engine, b, _chunks(ref_in)[:steps])
    assert sum(len(o) for o in out_a) > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert _same(out_a, out_b)
    # and the filter does something: the unfiltered stream differs
    c = made.create()
    if rate != FS:
        engine.session_set_input_rate(c, rate)
    assert not _same(out_a, _push(engine, c, _chunks(x, geo['n_in'])[:steps]))


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def test_learning_is_the_oracles_mean_and_applies_from_the_next_step(engine, made):
    steps, start, frames = 9, 1, 188
    x = _noisy((steps + 1) * T, stream=721, lead=1.6)
    chunks = _chunks(x)[:steps]

    def learn(busy=False):
        """(outputs, profiles and frames left after each step) of a session that learns from step `start` on"""
        sid = _denoising(engine, made)
        other = None
        if busy:
            other = _denoising(engine, made, 30.0, _profile(x))
            engine.session_denoise_learn(other, 50)
        buf = np.empty(engine.session_io_geometry(sid)['max_out'])
        outs, profiles, left = [], [], []
        for k, c in enumerate(chunks):
            if k == start:
                engine.session_denoise_learn(sid, frames)
                assert engine.session_noise_profile(sid)[1] == frames
            outs.append(engine.session_push(sid, c, buf).copy())
            if other is not None:
                engine.session_push(other, chunks[-1 - k])
            phi, n = engine.session_noise_profile(sid)
            profiles.append(phi)
            left.append(n)
        return outs, profiles, left

    outs, profiles, left = learn()
    # frames m of step k: [floor(k n / H), floor((k + 1) n / H))
    first = start * N // O.H
    want_left = [0] * start + [max(0, frames - ((k + 1) * N // O.H - first)) for k in range(start, steps)]
    print(f'frames left after each step: {left}')
    assert left == want_left
    done = want_left.index(0, start)                   # the step that adds the last frame
    want = O.frame_powers(x, first, frames).mean(axis=0)
    np.testing.assert_allclose(profiles[done], want, rtol=1e-12)
    assert not profiles[done - 1].any()
    # bitwise across runs and beside a busy session
    outs2, profiles2, left2 = learn(busy=True)
    assert left2 == left and all(np.array_equal(p, q) for p, q in zip(profiles, profiles2)) and _same(outs, outs2)
    # the learned profile applies from step done + 1 exactly: a session given it by hand in front of that step is bitwise the same
    hand = _denoising(engine, made)
    out_hand = _push(engine, hand, chunks, before=lambda k: k == done + 1 and engine.session_set_noise_profile(hand, profiles[done]))
    plain = _denoising(engine, made)
    out_plain = _push(engine, plain, chunks)
    assert _same(outs, out_hand)
    assert _same(outs[:done + 1], out_plain[:done + 1])
    assert not _same(outs[done + 1:], out_plain[done + 1:])


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
def test_settings_land_on_the_next_step_and_the_stream_is_the_oracles(engine, made, full_models, precision):
    from realtime_yukarin_b200.models import F0Converter
    engine.set_precision(precision)
    steps, j1, j2 = 7, 2, 4
    x = _noisy((steps + 1) * T, stream=731)
    chunks = _chunks(x)[:steps]
    phi = _profile(x)
    phi2 = 3.0 * phi

    def change(sid, k):
        if k == j1:
            engine.session_set_denoise(sid, 35.0)
        if k == j2:
            engine.session_set_noise_profile(sid, phi2)
    piped, blocking, never = (_denoising(engine, made, 10.0, phi) for _ in range(3))
    tickets = []
    for k, c in enumerate(chunks):                     # chunks in flight: nothing collected in between
        change(piped, k)
        tickets.append(engine.session_submit(piped, c))
        if k == 4:
            buf = np.empty(engine.session_io_geometry(piped)['max_out'])
            got = [engine.session_collect(piped, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
    out_blocking = _push(engine, blocking, chunks, before=lambda k: change(blocking, k))
    out_never = _push(engine, never, chunks)
    assert _same(got, out_blocking)
    assert _same(got[:j1], out_never[:j1]) and not _same(got[j1:], out_never[j1:])
    phi_now, left = engine.session_noise_profile(piped)
    assert np.array_equal(phi_now, phi2) and left == 0
    # the oracle: the filter with the same piecewise settings, then the reference's stream
    dn = O.DenoiseOracle(10.0, phi)
    stats = F0Converter(full_models['input_statistics_path'], full_models['target_statistics_path']).stats()
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    orc = opipe.StreamOracle(CFG, p1, p2, stats, buffer_time=T, extra=EXTRA, backend='torch')
    refs = []
    for k, c in enumerate(chunks):
        if k == j1:
            dn.set_reduction(35.0)
        if k == j2:
            dn.set_profile(phi2)
        refs.append(orc.push(dn.push(c)))
    assert [len(o) for o in got] == [len(r) for r in refs]
    y, r = np.concatenate(got), np.concatenate(refs)
    rmse, rms = _rmse(y, r), float(np.sqrt(np.mean(r ** 2)))
    print(f'{precision}: filtered stream vs StreamOracle on the oracle-filtered input: sample RMSE {rmse:.3e} (signal RMS {rms:.3e})')
    assert rms > 1e-2 and rmse <= TOL, rmse


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def test_the_filter_state_carries_over_groups_and_voice_switches(engine, made, full_models, second_voice_files):
    steps, out_at, back_at, switch_at = 9, 3, 6, 4
    x = _noisy((steps + 1) * T, stream=741)
    chunks = _chunks(x)[:steps]
    phi = _profile(x)
    # FP32: a member with the filter that leaves and joins again is bitwise its own session alone
    engine.set_precision('fp32')
    alone = _push(engine, _denoising(engine, made, 20.0, phi), chunks)
    a, b = _denoising(engine, made, 20.0, phi), made.create()
    gid = engine.group_create([a, b])
    made.gids.append(gid)
    bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(2)]
    got = []
    for k in range(steps):
        if k == out_at:
            engine.group_remove(gid, a)
        if k == back_at:
            engine.group_add(gid, a)
        members = engine.group_members(gid)
        if a in members:
            outs = engine.group_collect(gid, engine.group_submit(gid, [chunks[k] if s == a else chunks[-1 - k] for s in members]),
                                        bufs[:len(members)])
            got.append(outs[members.index(a)].copy())
        else:
            engine.group_collect(gid, engine.group_submit(gid, [chunks[-1 - k]]), bufs[:1])
            got.extend(_push(engine, a, [chunks[k]]))
    assert _same(got, alone)
    # FP16: within the group tolerance of the same member alone
    engine.set_precision('fp16')
    alone16 = _push(engine, _denoising(engine, made, 20.0, phi), chunks)
    a16, b16 = _denoising(engine, made, 20.0, phi), made.create()
    gid16 = engine.group_create([a16, b16])
    made.gids.append(gid16)
    got16 = [o[0].copy() for o in (engine.group_collect(gid16, engine.group_submit(gid16, [c, c]), bufs) for c in chunks)]
    err = _rmse(np.concatenate(got16), np.concatenate(alone16))
    print(f'fp16 group member with the filter vs alone: sample RMSE {err:.3e}')
    assert [len(o) for o in got16] == [len(o) for o in alone16] and err <= TOL
    # a voice switch keeps the filter's state: bitwise a session without the filter fed the whole-signal filtered input, switched alike
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    switched = _denoising(engine, made, 20.0, phi, voice=v1)
    reference = made.create(voice=v1)
    ref_in = _chunks(_filtered_input(engine, x[:steps * N], 20.0, phi))
    out_s = _push(engine, switched, chunks, before=lambda k: k == switch_at and engine.session_set_voice(switched, v2))
    out_r = _push(engine, reference, ref_in, before=lambda k: k == switch_at and engine.session_set_voice(reference, v2))
    assert _same(out_s, out_r)


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def _launch_windows(out_dir):
    """Child process of the launch-count test: returns (kernels the profiler saw, change of engine.launch_count) over 12 steps of a session
    without the filter fed the whole-signal filtered input (it runs the same kernels downstream: the silence gate picks the same
    stage-1 bodies) and of a session with the filter fed the input."""
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    _load(engine, synthetic.write_synthetic_models(out_dir / 'models', seed=0))
    engine.set_precision('fp16')
    steps = 12
    x = _noisy((steps + 1) * T, stream=751)
    phi = _profile(x)
    counts = {}
    for name, chunks in (('plain', _chunks(_filtered_input(engine, x[:steps * N], 20.0, phi))), ('filter', _chunks(x)[:steps])):
        sid = engine.session_create(_cfg())
        if name == 'filter':
            engine.session_denoise(sid)
            engine.session_set_noise_profile(sid, phi)
        counts[name] = _window(engine, out_dir, lambda: _push(engine, sid, chunks))
        engine.session_destroy(sid)
    return counts


def test_three_kernels_per_step_and_none_for_other_sessions(tmp_path):
    counts = _run_child(tmp_path, 'test_gpu_denoise', '_launch_windows')
    for name, (seen, counted) in counts.items():
        print(f'{name}: {counted} kernels counted over 12 steps, {seen} seen by the profiler')
        assert seen == counted, name
    assert counts['filter'][1] - counts['plain'][1] == 3 * 12


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 5
    x = _noisy((steps + 1) * T, stream=761)
    chunks = _chunks(x)[:steps]
    phi = _profile(x)
    sid, twin, plain = _denoising(engine, made, 20.0, phi), _denoising(engine, made, 20.0, phi), made.create()

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    outs = _push(engine, sid, chunks[:2])
    for db in (float('nan'), float('inf'), -0.5, 40.5):
        refused(lambda: engine.session_set_denoise(sid, db))
        refused(lambda: engine.denoise(x[:1000], db))
    for bad in (np.full(O.NB, np.nan), np.full(O.NB, np.inf), np.where(np.arange(O.NB) == 7, -1.0, phi)):
        refused(lambda: engine.session_set_noise_profile(sid, bad))
        refused(lambda: engine.denoise(x[:1000], 20.0, bad))
    refused(lambda: engine.session_denoise_learn(sid, frames=0))
    refused(lambda: engine.session_denoise(sid))               # ran a step
    refused(lambda: engine.session_denoise(99999))
    for call in (lambda: engine.session_set_denoise(plain, 10.0), lambda: engine.session_denoise_learn(plain, 10),
                 lambda: engine.session_set_noise_profile(plain, phi), lambda: engine.session_noise_profile(plain),
                 lambda: engine.session_set_denoise(99999, 10.0)):
        refused(call)
    assert np.array_equal(engine.session_noise_profile(sid)[0], phi) and engine.session_noise_profile(sid)[1] == 0
    assert engine.session_io_geometry(plain)['delay_in'] == 0
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_denoise(s)
        engine.session_denoise_learn(s, frames=60)
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with the filter')
    assert abs(grown) < 4.0


# ---- 8 ------------------------------------------------------------------------------------------------------------------------
def test_run_denoise_is_the_pipelines_denoise(engine, small_models, tmp_path):
    import yaml
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config
    from realtime_yukarin_b200.converter import YukarinConverter
    from realtime_yukarin_b200.worker import RealtimePipeline
    _load(engine, small_models)
    engine.set_precision('fp16')
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], extract_f0_mode='world')
    paths = {k: str(small_models[k]) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                               'stage1_config_path', 'stage2_model_path', 'stage2_config_path')}
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(dict(fields, **paths)))
    speech, _ = wave_io.read_wav(Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav')
    lead = np.zeros(FS, np.float32)
    clean = np.concatenate([lead, np.asarray(speech, np.float32)])
    noisy = clean + 0.02 * np.random.default_rng(771).standard_normal(len(clean)).astype(np.float32)
    wave_io.write_wav(tmp_path / 'noisy.wav', noisy, FS)
    args = ['--config_path', str(tmp_path / 'config.yaml'), '--wav_in', str(tmp_path / 'noisy.wav'), '--denoise', '20']
    run_mod.main(args + ['--wav_out', str(tmp_path / 'learn.wav'), '--learn_noise', '1', '--save_noise_profile', str(tmp_path / 'p.npy')])
    run_mod.main(args + ['--wav_out', str(tmp_path / 'loaded.wav'), '--noise_profile', str(tmp_path / 'p.npy')])
    saved = np.load(tmp_path / 'p.npy')
    assert saved.shape == (O.NB,) and saved.min() > 0
    config = Config.from_yaml(tmp_path / 'config.yaml')
    converter = YukarinConverter.make_yukarin_converter(**paths)
    param = converter.acoustic_converter.config.dataset.acoustic_param
    wave = wave_io.load_wave(tmp_path / 'noisy.wav', config.input_rate, engine=engine).wave

    def pipeline_run(**kw):
        pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, denoise=20.0, **kw)
        got = []
        try:
            for i in range(len(wave) // config.in_audio_chunk):
                got.append(pipe.process(wave[i * config.in_audio_chunk:(i + 1) * config.in_audio_chunk]))
            got.extend(pipe.drain())
            pipe.flush()
            profile = pipe.noise_profile()
        finally:
            pipe.close()
        return np.concatenate(got), profile

    def played(w):
        """the output chunks that carry sound: where the loop plays silence because nothing was ready yet depends on timing"""
        w = np.asarray(w)
        frames = w[:len(w) // config.out_audio_chunk * config.out_audio_chunk].reshape(-1, config.out_audio_chunk)
        return frames[np.any(frames != 0, axis=1)]

    mine, (phi, left) = pipeline_run(learn_noise=1.0)
    assert left == 0 and np.array_equal(phi, saved)
    # the learned profile is the mean over frames 0 .. 187 of the input (a session analyses from its first sample on)
    np.testing.assert_allclose(phi, O.frame_powers(wave, 0, 188).mean(axis=0), rtol=1e-12)
    run_learn = wave_io.load_wave(tmp_path / 'learn.wav', FS, engine=engine).wave
    assert len(played(mine)) >= 10 and np.array_equal(played(run_learn), played(mine))
    mine_loaded, (phi_loaded, _) = pipeline_run(noise_profile=saved)
    assert np.array_equal(phi_loaded, saved)
    run_loaded = wave_io.load_wave(tmp_path / 'loaded.wav', FS, engine=engine).wave
    assert np.array_equal(played(run_loaded), played(mine_loaded))
