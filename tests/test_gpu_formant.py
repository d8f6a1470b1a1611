"""The per-session formant ratio (ryk_session_set_formant) and the per-op warp (ryk_stage2_convert_formant), at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), FP16, base-64 synthetic models.

  * a session that never sets a ratio, or sets 1, is bitwise what it was, with the same kernels; ratio 1 per op is bitwise the plain call;
  * the kernel's warp is exp(numpy.interp(k / r, arange(513), log(plain output))) and moves a peak from bin p to about p r;
  * a set takes effect exactly at the step it was submitted before, with chunks in flight; the stream is the oracle's stream;
  * group members keep their own ratios, through ryk_group_remove / _add;
  * refused calls change nothing; create / set / destroy cycles return their memory; run.py --formant is RealtimePipeline(formant=).
"""
import math
from pathlib import Path

import numpy as np
import pytest

from oracle import nets as onets
from realtime_yukarin_b200.engine import RykError

from .formant_oracle import FormantStreamOracle, formant_warp
from .test_gpu_f0_control import (CFG, EXTRA, FS, TOL, T, _cfg, _new_voice, _push, _same, _speech, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_headline_parity import _rmse, _waveform_spectral_distance
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

NB = 513
RATIOS = [0.5, 0.8, 2 ** (-3 / 12), 2 ** (5 / 12), 2.0]


def _envelopes(engine, stream=601, steps=2):
    """(T, 513) float32 spectral envelopes of synthetic speech, from the engine's own analysis"""
    x = np.concatenate(_speech(steps, stream=stream))
    f = engine.world_analyze(x, FS, 5.0, 71.0, 800.0, 1024, 8, 0.466)
    return np.ascontiguousarray(f['sp'], np.float32) + np.float32(1e-16)


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_nothing_moves_by_default(engine, made):
    steps = 14
    chunks = _speech(steps, stream=601)
    a, b = made.create(), made.create()
    assert engine.session_get_formant(a) == 1.0
    engine.session_set_formant(b, ratio=1.0)
    assert engine.session_get_formant(b) == 1.0
    before = engine.launch_count
    out_a = _push(engine, a, chunks)
    count_a = engine.launch_count - before
    before = engine.launch_count
    out_b = _push(engine, b, chunks)
    count_b = engine.launch_count - before
    assert _same(out_a, out_b)
    assert sum(len(o) for o in out_a) > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    print(f'{count_a / steps:.1f} kernels per step, {count_b / steps:.1f} with the ratio set to 1')
    assert count_a == count_b
    sp = _envelopes(engine)
    assert np.array_equal(engine.stage2_convert(sp, 1.0), engine.stage2_convert(sp))


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
def test_the_kernels_warp_is_the_oracles_warp(engine, made):
    sp = _envelopes(engine, stream=611)
    plain = engine.stage2_convert(sp)
    logs = np.log(plain.astype(np.float64))
    k = np.arange(NB)
    for r in RATIOS:
        got = engine.stage2_convert(sp, r)
        want = np.exp(np.stack([np.interp(k / r, k, row) for row in logs]))
        np.testing.assert_allclose(got, want, rtol=1e-5, err_msg=f'ratio {r}')
        assert not np.array_equal(got, plain)
        # the oracle's writing of the warp on the same network output
        np.testing.assert_allclose(got, np.exp(formant_warp(logs[:, :-1].astype(np.float32), r)), rtol=1e-5, err_msg=f'ratio {r}')
    # the peak of a sharp local maximum at bin p moves to round(p r) +- 1
    moved = 0
    for r in (0.8, 1.25):
        got = np.log(engine.stage2_convert(sp, r).astype(np.float64))
        for t in range(0, len(logs), 7):
            L = logs[t]
            for p in range(45, 200):
                win = L[p - 5:p + 6]
                if np.argmax(win) != 5 or np.partition(win, -2)[-2] > L[p] - 0.05:
                    continue
                q = round(p * r)
                ref = formant_warp(L[None, :-1].astype(np.float32), r)[0]
                if abs(q - 3 + int(np.argmax(ref[q - 3:q + 4])) - q) > 1:
                    continue                       # a neighbour close to the peak: sampling may put the maximum two bins off
                assert abs(q - 3 + int(np.argmax(got[t, q - 3:q + 4])) - q) <= 1, (r, t, p)
                moved += 1
    print(f'{moved} sharp peaks moved to round(p r) +- 1')
    assert moved >= 5


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def test_a_set_lands_on_the_step_it_was_submitted_before(engine, made):
    steps, j, ratio = 5, 3, 1.3
    chunks = _speech(steps, stream=621)
    piped, blocking, never, fresh = made.create(), made.create(), made.create(), made.create()
    tickets = []
    for k in range(steps):                               # five chunks in flight, nothing collected in between
        if k == j:
            engine.session_set_formant(piped, ratio=ratio)
        tickets.append(engine.session_submit(piped, chunks[k]))
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    out_piped = [engine.session_collect(piped, t, buf).copy() for t in tickets]
    out_blocking = _push(engine, blocking, chunks, before=lambda k: k == j and engine.session_set_formant(blocking, ratio=ratio))
    out_never = _push(engine, never, chunks)
    assert engine.session_get_formant(piped) == ratio
    assert _same(out_piped, out_blocking)
    assert _same(out_piped[:j], out_never[:j])
    assert not _same(out_piped[j:], out_never[j:])
    # a set on a fresh session applies from step 0
    engine.session_set_formant(fresh, ratio=ratio)
    out_fresh = _push(engine, fresh, chunks)
    assert not _same(out_fresh, out_never)


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['octave up', 'pitch and formant +4', 'down from step 0'])
def test_the_stream_is_the_oracles_stream(engine, made, full_models, case):
    from realtime_yukarin_b200.models import F0Converter
    steps = 8
    j = 0 if case == 'down from step 0' else 3
    chunks = _speech(steps, stream=631)
    stats = F0Converter(full_models['input_statistics_path'], full_models['target_statistics_path']).stats()
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    orc = FormantStreamOracle(CFG, p1, p2, stats, buffer_time=T, extra=EXTRA, backend='torch')
    sid, plain = made.create(), made.create()
    new_stats, ratio = stats, {'octave up': 2.0, 'pitch and formant +4': 2 ** (4 / 12), 'down from step 0': 0.85}[case]

    def change():
        if case == 'pitch and formant +4':
            engine.session_set_f0_map(sid, semitones=4)
            engine.session_set_formant(sid, semitones=4)
        else:
            engine.session_set_formant(sid, ratio=ratio)
    if case == 'pitch and formant +4':
        new_stats = (stats[0], stats[1], stats[2] + 4 * math.log(2.0) / 12, stats[3])
    outs = _push(engine, sid, chunks, before=lambda k: k == j and change())
    assert engine.session_get_formant(sid) == pytest.approx(ratio, rel=1e-15)
    refs = []
    for k, c in enumerate(chunks):
        if k == j:
            orc.f0_stats, orc.formant_ratio = new_stats, ratio
        refs.append(orc.push(c))
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse, rms, lsd = _rmse(y, r), float(np.sqrt(np.mean(r ** 2))), _waveform_spectral_distance(y, r)
    print(f'formant ratio {ratio:.4f} from step {j} ({case}): {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), '
          f'log-STFT distance {lsd:.3e}')
    assert rms > 1e-2
    assert rmse <= TOL, rmse
    assert lsd <= 0.1, lsd
    unchanged = _push(engine, plain, chunks)
    moved = _rmse(np.concatenate(outs[j:]), np.concatenate(unchanged[j:]))
    print(f'steps {j}.. moved by sample RMSE {moved:.3e} from the unchanged stream')
    # the change is far outside the distance to the oracle.  An upward warp alone moves little of the synthetic voice's energy: its
    # harmonics sit low, where the envelope is nearly flat (an octave up moves the stream by about 6e-3 RMSE, 250 times the match)
    assert moved > 100 * rmse
    if case != 'octave up':
        assert moved > 10 * TOL


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def test_group_members_keep_their_own_ratios(engine, made, full_models, second_voice_files):
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    steps, j, out_at, back_at, ratio = 9, 2, 5, 7, 0.8
    xs = {name: _speech(steps, stream=640 + i) for i, name in enumerate('abc')}

    def change_a(sid, k, change):
        if change and k == j:
            engine.session_set_formant(sid, ratio=ratio)

    a = made.create(voice=v1)
    alone_a = _push(engine, a, xs['a'], before=lambda k: change_a(a, k, True))

    def grouped(change):
        """a, b (voice 1) and c (voice 2) in one group; a leaves before step out_at and joins again before step back_at"""
        a, b, c = made.create(voice=v1), made.create(voice=v1), made.create(voice=v2)
        gid = engine.group_create([a, b, c])
        made.gids.append(gid)
        bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(3)]
        got = {name: [] for name in 'abc'}
        for k in range(steps):
            if k == out_at:
                engine.group_remove(gid, a)
                assert engine.session_get_formant(a) == (ratio if change else 1.0)
            if k == back_at:
                engine.group_add(gid, a)
                assert engine.session_get_formant(a) == (ratio if change else 1.0)
            change_a(a, k, change)
            members = engine.group_members(gid)
            names = ['abc'[(a, b, c).index(s)] for s in members]
            outs = engine.group_collect(gid, engine.group_submit(gid, [xs[n][k] for n in names]), bufs[:len(members)])
            for n, o in zip(names, outs):
                got[n].append(o.copy())
            if 'a' not in names:
                got['a'].extend(_push(engine, a, [xs['a'][k]]))
        assert engine.session_get_formant(b) == engine.session_get_formant(c) == 1.0
        return got

    untouched, changed = grouped(False), grouped(True)
    for n in 'bc':
        assert _same(changed[n], untouched[n]), n
    assert _same(changed['a'][:j], untouched['a'][:j])
    assert not _same(changed['a'][j:], untouched['a'][j:])
    assert [len(o) for o in changed['a']] == [len(o) for o in alone_a]
    err = _rmse(np.concatenate(changed['a']), np.concatenate(alone_a))
    print(f'member a with ratio {ratio} from step {j}: grouped (alone for steps {out_at}..{back_at - 1}) vs alone, sample RMSE {err:.3e}')
    assert err <= TOL, err
    moved = _rmse(np.concatenate(changed['a'][j:]), np.concatenate(untouched['a'][j:]))
    print(f'member a moved by sample RMSE {moved:.3e} from step {j} on')
    assert moved > 100 * err                             # far outside its distance to the ungrouped run (see the oracle test)


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 6
    chunks = _speech(steps, stream=651)
    sid, twin = made.create(), made.create()
    engine.session_set_formant(sid, ratio=1.1)
    engine.session_set_formant(twin, ratio=1.1)

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    outs = _push(engine, sid, chunks[:2])
    bad = (float('nan'), float('inf'), -float('inf'), 0.0, -1.0, 0.49, 2.01)
    for r in bad:
        refused(lambda: engine.session_set_formant(sid, ratio=r))
    refused(lambda: engine.session_set_formant(99999, ratio=1.2))
    refused(lambda: engine.session_get_formant(99999))
    assert engine.session_get_formant(sid) == 1.1
    sp = _envelopes(engine, stream=652, steps=1)
    for r in bad:
        with pytest.raises(RykError):
            engine.stage2_convert(sp, r)
    for r in (0.5, 2.0):                                 # the ends of the range are allowed
        engine.session_set_formant(twin, ratio=r)
        assert engine.session_get_formant(twin) == r
    engine.session_set_formant(twin, ratio=1.1)
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    # create / set / push / destroy
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_set_formant(s, semitones=(cycle % 5) - 2)
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with a formant ratio')
    assert abs(grown) < 4.0


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def test_run_formant_is_the_pipelines_formant(engine, small_models, tmp_path):
    import yaml
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200 import wave_io
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
    wav_in = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
    outs = {}
    for semis in (3, 0):
        run_mod.main(['--config_path', str(tmp_path / 'config.yaml'), '--wav_in', str(wav_in), '--wav_out', str(tmp_path / f'run{semis}.wav'),
                      '--formant', str(semis)])
        outs[semis] = wave_io.load_wave(tmp_path / f'run{semis}.wav', FS, engine=engine).wave
    config = Config.from_yaml(tmp_path / 'config.yaml')
    converter = YukarinConverter.make_yukarin_converter(**paths)
    pipe = RealtimePipeline(config, acoustic_param=converter.acoustic_converter.config.dataset.acoustic_param, engine=engine, formant=3)
    wave = wave_io.load_wave(wav_in, config.input_rate, engine=engine).wave
    got = []
    try:
        n = len(wave) // config.in_audio_chunk
        for i in range(n):
            got.append(pipe.process(wave[i * config.in_audio_chunk:(i + 1) * config.in_audio_chunk]))
        got.extend(pipe.drain())
    finally:
        pipe.close()
    wave_io.write_wav(tmp_path / 'pipe.wav', np.concatenate(got), config.output_rate)
    mine = wave_io.load_wave(tmp_path / 'pipe.wav', FS, engine=engine).wave

    def played(w):
        """the output chunks that carry sound: where the loop plays silence because nothing was ready yet depends on timing"""
        w = np.asarray(w)
        frames = w[:len(w) // config.out_audio_chunk * config.out_audio_chunk].reshape(-1, config.out_audio_chunk)
        return frames[np.any(frames != 0, axis=1)]
    assert len(played(mine)) >= 10
    assert np.array_equal(played(outs[3]), played(mine))
    assert played(outs[0]).shape != played(mine).shape or not np.array_equal(played(outs[0]), played(mine))
