"""The per-session f0 map (ryk_session_set_f0_map), the speaker's log-f0 statistics measured on the device (ryk_session_f0_measure /
_f0_measured) and follow mode (ryk_session_f0_follow), at the headline configuration: 0.3 s chunks, extras (0, 0.5, 0), FP16, base-64
synthetic models.

  * a session that does not use them, or that sets its voice's own values, is bitwise what it was; measuring adds one kernel per step;
  * the measurement is numpy's FP64 mean / std of ln f0 over the voiced frames of the same analysis, bitwise reproducible;
  * a set takes effect exactly at the step it was submitted before, with chunks in flight; the map is the oracle's map;
  * follow mode is bitwise a host that reads the measurement and sets the map before every step;
  * group members keep their own maps through ryk_group_remove; other sessions of the voice and the voice itself are untouched;
  * refused calls change nothing; create / measure / follow / destroy cycles return their memory; run.py writes a statistics file.
"""
import math
from pathlib import Path

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import RykError, SessionConfig

from .test_gpu_headline_parity import _rmse, _waveform_spectral_distance
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()
FS, T = 24000, 0.3
N = round(T * FS)
EXTRA = (0.0, 0.5, 0.0)
TOL = 1e-3                      # sample RMSE of tests/test_gpu_headline_parity.py and tests/test_gpu_group_membership.py


def _cfg():
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                         encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                         vocoder_buffer_size=1024)


def _chunks(x):
    return [np.ascontiguousarray(x[k * N:(k + 1) * N], np.float32) for k in range(len(x) // N)]


def _speech(steps, stream):
    return _chunks(synthetic.synthetic_speech((steps + 1) * T, stream=stream))[:steps]


def _tone(steps, hz=150.0):
    """a steady harmonic tone: voiced, with (almost) one f0"""
    t = np.arange(steps * N) / FS
    return _chunks(0.2 * sum(np.sin(2 * np.pi * h * hz * t) / h for h in range(1, 11)))


SILENCE = np.zeros(N, np.float32)


class _Sessions:
    """Sessions of a test on the shared engine, destroyed (groups first, voices last) whatever failed."""

    def __init__(self, engine):
        self.engine, self.sids, self.gids, self.voices = engine, [], [], []

    def create(self, voice=0, measure=False, follow=None, sd_floor=None, f0_method=None):
        e = self.engine
        prev = e.f0_method
        if f0_method:
            e.set_f0_method(f0_method)
        try:
            sid = e.session_create(_cfg(), voice=voice)
        finally:
            e.set_f0_method(prev)
        self.sids.append(sid)
        if measure or follow is not None:
            e.session_f0_measure(sid)
        if follow is not None:
            e.session_f0_follow(sid, True, min_voiced_frames=follow, **({} if sd_floor is None else {'sd_floor': sd_floor}))
        return sid

    def close(self):
        e = self.engine
        for items, destroy in ((self.gids, e.group_destroy), (self.sids, e.session_destroy), (self.voices, e.voice_destroy)):
            while items:
                destroy(items.pop())
        e.set_f0_method('dio')
        e.set_precision('fp16')


@pytest.fixture
def made(engine, full_models):
    _load(engine, full_models)
    engine.set_precision('fp16')
    m = _Sessions(engine)
    yield m
    m.close()


def _push(engine, sid, chunks, before=None, first=0):
    """blocking pushes; before(k) runs in front of the push of step k"""
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    outs = []
    for k, c in enumerate(chunks, first):
        if before:
            before(k)
        outs.append(engine.session_push(sid, c, buf).copy())
    return outs


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _log_f0(engine, chunks, method='dio'):
    """ln f0 (FP64) of the voiced frames of the per-op analysis of each chunk: the kernels the session's analysis runs"""
    prev = engine.f0_method
    engine.set_f0_method(method)
    try:
        logs = []
        for c in chunks:
            f = engine.world_analyze(c, FS, 5.0, 71.0, 800.0, 1024, 8, 0.466)
            v = f['voiced'] & (f['f0'] > 0)
            logs.append(np.log(f['f0'][v].astype(np.float64)))
        return np.concatenate(logs)
    finally:
        engine.set_f0_method(prev)


def _check_measured(got, logs):
    n, mean, std = got
    assert n == len(logs)
    if n == 0:
        assert (mean, std) == (0.0, 0.0)
        return
    assert abs(mean - logs.mean()) <= 1e-12, (mean, logs.mean())
    want = logs.std() if n >= 2 else 0.0
    assert abs(std - want) <= 1e-10 * max(want, 1e-300), (std, want)


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def test_nothing_moves_by_default(engine, made, full_models):
    from realtime_yukarin_b200.models import F0Converter
    steps = 14
    chunks = _speech(steps, stream=501)
    a, b = made.create(), made.create(measure=True)
    stats = F0Converter(full_models['input_statistics_path'], full_models['target_statistics_path']).stats()
    assert tuple(engine.session_get_f0_map(a).values()) == stats
    engine.session_set_f0_map(b, **engine.session_get_f0_map(b))
    assert engine.session_get_f0_map(b) == engine.session_get_f0_map(a)
    before = engine.launch_count
    out_a = _push(engine, a, chunks)
    count_a = engine.launch_count - before
    before = engine.launch_count
    out_b = _push(engine, b, chunks)
    count_b = engine.launch_count - before
    assert _same(out_a, out_b)
    assert sum(len(o) for o in out_a) > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    print(f'{count_a / steps:.1f} kernels per step, {count_b / steps:.1f} with the measuring kernel')
    # the measuring kernel, once per step, on top of the count tests/test_gpu_launch_count.py checks against the profiler
    assert count_b - count_a == steps
    assert engine.session_f0_measured(b)[0] > 0


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('method', ['dio', 'harvest'])
def test_measurement_is_numpy_on_the_same_frames(engine, made, method):
    steps = 10
    chunks = _speech(steps, stream=511)
    sid = made.create(measure=True, f0_method=method)
    assert engine.session_f0_measured(sid) == (0, 0.0, 0.0)
    _push(engine, sid, chunks[:4])
    logs4 = _log_f0(engine, chunks[:4], method)
    assert len(logs4) > 100
    _check_measured(engine.session_f0_measured(sid), logs4)
    _push(engine, sid, chunks[4:])
    got = engine.session_f0_measured(sid)
    _check_measured(got, _log_f0(engine, chunks, method))
    # the oracle's analysis of the same chunks, at the tolerance of the f0 parity tests (voiced decisions exact, f0 to 1e-6 relative)
    pc = opipe.PathConfig(f0_method=method)
    ref = []
    for c in chunks[:6]:
        f = opipe.extract_features(c, pc)
        ref.append(np.log(f['f0'].ravel()[f['voiced'].ravel()].astype(np.float64)))
    ref = np.concatenate(ref)
    dev = _log_f0(engine, chunks[:6], method)
    assert len(ref) == len(dev) and abs(ref.mean() - dev.mean()) <= 1e-6 and abs(ref.std() - dev.std()) <= 2e-6
    # reset: from the next step on
    engine.session_f0_measure_reset(sid)
    assert engine.session_f0_measured(sid) == (0, 0.0, 0.0)
    more = _speech(3, stream=512)
    _push(engine, sid, more)
    _check_measured(engine.session_f0_measured(sid), _log_f0(engine, more, method))


def test_silence_counts_nothing_and_runs_are_bitwise_equal(engine, made):
    quiet = made.create(follow=1)
    plain = made.create()
    silent = [SILENCE] * 3
    assert _same(_push(engine, quiet, silent), _push(engine, plain, silent))
    assert engine.session_f0_measured(quiet) == (0, 0.0, 0.0)
    assert engine.session_get_f0_map(quiet) == engine.session_get_f0_map(plain)
    # the same stream twice, the second time beside a busy session: bitwise the same triple after every step
    steps = 8
    chunks = _speech(steps, stream=513)
    other = _speech(steps, stream=514)
    first, busy = made.create(measure=True), made.create()
    triples = []
    _push(engine, first, chunks, before=lambda k: k and triples.append(engine.session_f0_measured(first)))
    triples.append(engine.session_f0_measured(first))
    second = made.create(measure=True)
    buf = np.empty(engine.session_io_geometry(second)['max_out'])
    again = []
    for k in range(steps):
        tb = engine.session_submit(busy, other[k])
        ts = engine.session_submit(second, chunks[k])
        again.append(engine.session_f0_measured(second))
        engine.session_collect(second, ts, buf)
        engine.session_collect(busy, tb, buf)
    assert len(triples) == steps and triples == again
    assert triples[-1][0] > triples[0][0] > 0


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def test_a_set_lands_on_the_step_it_was_submitted_before(engine, made):
    steps, j = 5, 3
    chunks = _speech(steps, stream=521)
    new = dict(in_mean=math.log(120.0), in_std=0.25, target_mean=math.log(320.0), target_std=0.15)
    piped, blocking, never = made.create(), made.create(), made.create()
    tickets = []
    for k in range(steps):                               # five chunks in flight, nothing collected in between
        if k == j:
            engine.session_set_f0_map(piped, **new)
        tickets.append(engine.session_submit(piped, chunks[k]))
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    out_piped = [engine.session_collect(piped, t, buf).copy() for t in tickets]
    out_blocking = _push(engine, blocking, chunks, before=lambda k: k == j and engine.session_set_f0_map(blocking, **new))
    out_never = _push(engine, never, chunks)
    assert engine.session_get_f0_map(piped) == new
    assert _same(out_piped, out_blocking)
    assert _same(out_piped[:j], out_never[:j])
    assert not _same(out_piped[j:], out_never[j:])        # and the new map is audible from step j on


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['new statistics', 'octave up'])
def test_the_map_is_the_oracles_map(engine, made, full_models, case):
    from realtime_yukarin_b200.models import F0Converter
    steps, j = 8, 3
    chunks = _speech(steps, stream=531)
    stats = F0Converter(full_models['input_statistics_path'], full_models['target_statistics_path']).stats()
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    orc = opipe.StreamOracle(CFG, p1, p2, stats, buffer_time=T, extra=EXTRA, backend='torch')
    sid, plain = made.create(), made.create()
    if case == 'octave up':
        new_stats = (stats[0], stats[1], stats[2] + math.log(2.0), stats[3])
        change = lambda: engine.session_set_f0_map(sid, semitones=12)
    else:
        new_stats = (math.log(130.0), 0.3, math.log(210.0), 0.12)
        change = lambda: engine.session_set_f0_map(sid, *new_stats)
    outs = _push(engine, sid, chunks, before=lambda k: k == j and change())
    assert tuple(engine.session_get_f0_map(sid).values()) == pytest.approx(new_stats, rel=1e-15)
    refs = []
    for k, c in enumerate(chunks):
        if k == j:
            orc.f0_stats = new_stats
        refs.append(orc.push(c))
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse, rms, lsd = _rmse(y, r), float(np.sqrt(np.mean(r ** 2))), _waveform_spectral_distance(y, r)
    print(f'f0 map changed at step {j} ({case}): {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), log-STFT distance {lsd:.3e}')
    assert rms > 1e-2
    assert rmse <= TOL, rmse
    assert lsd <= 0.1, lsd
    unchanged = np.concatenate(_push(engine, plain, chunks))
    assert _rmse(y, unchanged) > 10 * TOL                # the change is far outside the tolerance it is matched to


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def _follow_by_hand(engine, made, chunks, min_voiced, sd_floor):
    """(outputs of the following session, of the session whose map the host sets from the measurement, of an untouched one, and the
    step at which the count reached min_voiced)"""
    measuring = made.create(measure=True)
    following = made.create(follow=min_voiced, sd_floor=sd_floor)
    by_hand, plain = made.create(), made.create()
    reached, floored = [], []

    def host_rule(k):
        _push(engine, measuring, [chunks[k]])
        n, mean, std = engine.session_f0_measured(measuring)      # includes the frames of chunk k
        if n >= min_voiced:
            reached.append(k)
            floored.append(std < sd_floor)
            engine.session_set_f0_map(by_hand, in_mean=mean, in_std=max(std, sd_floor))
    out_hand = _push(engine, by_hand, chunks, before=host_rule)
    out_follow = _push(engine, following, chunks)
    out_plain = _push(engine, plain, chunks)
    assert engine.session_f0_measured(following) == engine.session_f0_measured(measuring)
    return out_follow, out_hand, out_plain, reached, floored


def test_follow_mode_is_a_host_that_sets_the_measurement_every_step(engine, made):
    speech = _speech(18, stream=541)
    chunks = speech[:5] + [SILENCE] * 3 + speech[5:]                 # 21 steps
    out_follow, out_hand, out_plain, reached, floored = _follow_by_hand(engine, made, chunks, min_voiced=140, sd_floor=0.05)
    assert 0 < reached[0] < 5 and reached == list(range(reached[0], len(chunks))), reached
    assert not any(floored)
    for k, (f, h) in enumerate(zip(out_follow, out_hand)):
        assert np.array_equal(f, h), k
    assert _same(out_follow[:reached[0]], out_plain[:reached[0]])     # the voice's values until the count is reached
    assert not _same(out_follow[reached[0]:], out_plain[reached[0]:])


def test_follow_mode_floors_a_monotone_speaker(engine, made):
    chunks = _tone(12)
    out_follow, out_hand, out_plain, reached, floored = _follow_by_hand(engine, made, chunks, min_voiced=100, sd_floor=0.05)
    assert reached and all(floored), (reached, floored)               # the tone's own std is far below the floor
    for k, (f, h) in enumerate(zip(out_follow, out_hand)):
        assert np.array_equal(f, h) and np.isfinite(f).all(), k
    assert not _same(out_follow, out_plain)


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def second_voice_files(tmp_path_factory):
    return synthetic.write_synthetic_models(tmp_path_factory.mktemp('f0_voice2'), seed=41)


def _new_voice(engine, made, paths):
    from realtime_yukarin_b200.models import load_voice
    v = engine.voice_create()
    made.voices.append(v)
    load_voice(engine, v, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                   'target_statistics_path')})
    return v


def test_group_members_keep_their_own_maps(engine, made, full_models, second_voice_files):
    v1, v2 = _new_voice(engine, made, full_models), _new_voice(engine, made, second_voice_files)
    grouped_steps, alone_steps, j = 6, 3, 3
    steps = grouped_steps + alone_steps
    xs = {name: _speech(steps, stream=550 + i) for i, name in enumerate('abcd')}
    map_a = dict(in_mean=math.log(130.0), in_std=0.15)

    def trio():
        a, b, c = made.create(voice=v1), made.create(voice=v1, follow=100), made.create(voice=v2)
        engine.session_set_f0_map(a, **map_a)
        return a, b, c

    def change_a(sid, k):
        if k == j:
            engine.session_set_f0_map(sid, semitones=2)

    # every stream alone, on a quiet engine
    a, b, c = trio()
    alone = {'a': _push(engine, a, xs['a'], before=lambda k: change_a(a, k)), 'b': _push(engine, b, xs['b']),
             'c': _push(engine, c, xs['c'])}
    measured_alone = engine.session_f0_measured(b)
    d = made.create(voice=v1)
    alone['d'] = _push(engine, d, xs['d'])
    map_d = engine.session_get_f0_map(d)
    # the same streams as members of one mixed-voice group, with a fourth session of voice 1 running beside it
    a, b, c = trio()
    d = made.create(voice=v1)
    gid = engine.group_create([a, b, c])
    made.gids.append(gid)
    with pytest.raises(RykError):
        engine.f0_set_stats(5.0, 0.2, 5.5, 0.2, voice=v1)            # the voice stays locked; the sessions' maps are their own
    bufs = [np.empty(engine.session_io_geometry(a)['max_out']) for _ in range(3)]
    got = {name: [] for name in 'abcd'}
    for k in range(steps):
        members = engine.group_members(gid)
        if k == grouped_steps:
            engine.group_remove(gid, a)
            members = engine.group_members(gid)
            assert members == [b, c]
        change_a(a, k)                                              # at step j: a set on a group member
        names = ['abc'[(a, b, c).index(s)] for s in members]
        outs = engine.group_collect(gid, engine.group_submit(gid, [xs[n][k] for n in names]), bufs[:len(members)])
        for n, o in zip(names, outs):
            got[n].append(o.copy())
        if k >= grouped_steps:
            got['a'].extend(_push(engine, a, [xs['a'][k]]))
        got['d'].extend(_push(engine, d, [xs['d'][k]]))
    assert engine.session_get_f0_map(a)['target_mean'] == pytest.approx(map_d['target_mean'] + 2 * math.log(2.0) / 12, rel=1e-15)
    assert engine.session_get_f0_map(d) == map_d
    assert _same(got['d'], alone['d'])                              # a session of the voice that never set anything: bitwise
    assert engine.session_f0_measured(b) == measured_alone          # stage 1 is the member's own, grouped or not
    for n in 'abc':
        assert [len(o) for o in got[n]] == [len(o) for o in alone[n]], n
        err = _rmse(np.concatenate(got[n]), np.concatenate(alone[n]))
        print(f'member {n}: grouped (alone from step {grouped_steps} on for a) vs alone, sample RMSE {err:.3e}')
        assert err <= TOL, (n, err)
    assert _rmse(np.concatenate(got['a']), np.concatenate(got['b'])) > 10 * TOL


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    steps = 6
    chunks = _speech(steps, stream=561)
    sid, twin, measuring = made.create(), made.create(), made.create(measure=True)
    good = engine.session_get_f0_map(sid)
    nan, inf = float('nan'), float('inf')

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    outs = _push(engine, sid, chunks[:2])
    for bad in (dict(in_mean=nan), dict(target_mean=inf), dict(in_std=0.0), dict(in_std=-0.1), dict(target_std=0.0), dict(target_std=nan)):
        refused(lambda: engine.session_set_f0_map(sid, **bad))
    refused(lambda: engine.session_f0_follow(sid, True))                      # follow without measuring
    refused(lambda: engine.session_f0_measure(sid))                           # measuring on a session that has run a step
    refused(lambda: engine.session_f0_measured(sid))
    refused(lambda: engine.session_f0_measure_reset(sid))
    refused(lambda: engine.session_f0_follow(measuring, True, min_voiced_frames=0))
    refused(lambda: engine.session_f0_follow(measuring, True, sd_floor=nan))
    refused(lambda: engine.session_f0_follow(measuring, True, sd_floor=0.0))
    for call in (engine.session_get_f0_map, engine.session_set_f0_map, engine.session_f0_measure, engine.session_f0_measured,
                 engine.session_f0_measure_reset, engine.session_f0_follow):
        refused(lambda: call(99999))                                          # unknown session
    assert engine.session_get_f0_map(sid) == good
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    assert _same(_push(engine, measuring, chunks), outs)                      # its refused follow calls left it measuring only
    # create / measure / follow / push / destroy
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_f0_measure(s)
        engine.session_f0_follow(s, True, min_voiced_frames=30)
        engine.session_set_f0_map(s, semitones=1)
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        assert engine.session_f0_measured(s)[0] > 30
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 measuring session cycles')
    assert abs(grown) < 4.0


# ---- 8 ------------------------------------------------------------------------------------------------------------------------
def test_run_measures_the_input_statistics_of_a_wav(engine, small_models, tmp_path):
    import yaml
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200 import wave_io
    from realtime_yukarin_b200.models import F0Converter
    _load(engine, small_models)
    engine.set_precision('fp16')
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], extract_f0_mode='world')
    paths = {k: str(small_models[k]) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                               'stage1_config_path', 'stage2_model_path', 'stage2_config_path')}
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(dict(fields, **paths)))
    wav_in = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
    out = tmp_path / 'measured_statistics.npy'
    n = run_mod.run(tmp_path / 'config.yaml', wav_in=wav_in, wav_out=tmp_path / 'out.wav', engine=engine, depth=2,
                    measure_input_statistics=out)
    wave = wave_io.load_wave(wav_in, FS, engine=engine).wave
    assert n == len(wave) // N and n >= 10
    logs = _log_f0(engine, _chunks(np.asarray(wave, np.float32))[:n])
    assert len(logs) > 100
    f0c = F0Converter(out, small_models['target_statistics_path'])            # the file drops into input_statistics_path
    assert abs(f0c.input_mean - logs.mean()) <= 1e-12
    assert abs(f0c.input_var - logs.var()) <= 1e-9 * logs.var()
    d = np.load(str(out), allow_pickle=True).item()
    assert (d['mean'], d['var']) == (f0c.input_mean, f0c.input_var)
