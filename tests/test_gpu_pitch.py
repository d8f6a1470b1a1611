"""The pitch correction of a streaming session (ryk_session_pitch_correct and its calls) and the whole-signal ryk_pitch_correct, at the
headline configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models, and with a decode extra.

  1. ryk_pitch_correct is the FP64 oracle (tests/pitch_oracle.py) to 1e-12 relative, with the same note choices except at a decision
     boundary (reported), and bitwise repeatable;
  2. amount 0 is a session without the stage bit for bit; the stage adds one kernel per step and none to other sessions;
  3. the rows a session with the stage appends to its decode window are ryk_pitch_correct of those a session without it appends,
     bitwise, at the headline extras and with a decode extra; its output re-analysed sits on scale notes;
  4. a setting change lands on the next submitted step;  5. group members are the session alone; a voice switch keeps the glide state;
  6. snapshot / restore mid-stream continues bitwise; a session without the stage writes the same sections as before;
  7. refusals change nothing; enable / destroy cycles return memory;  8. run.py --autotune is RealtimePipeline(pitch_correct=...).
The session's decode-window rows are read from its snapshots (DWF0 sections): the state a moved session carries.
"""
import math
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import PITCH_SCALES, RykError, describe_snapshot

from . import pitch_oracle as P
from .test_gpu_f0_control import (EXTRA, FS, N, T, _cfg, _new_voice, _push, _same, _speech, _tone, made,  # noqa: F401
                                  second_voice_files)
from .test_gpu_launch_count import _run_child, _window
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

HOP = 5.0
MAJOR = PITCH_SCALES['major']
SETTINGS = dict(key='D', scale='major', a4_hz=442.0, retune_ms=30.0, amount=1.0)


def _sections(blob):
    """[(tag, payload)] of a snapshot blob"""
    out, at = [], 32
    while at < len(blob):
        tag = blob[at:at + 4].decode('ascii')
        n = int.from_bytes(blob[at + 8:at + 16], 'little')
        out.append((tag, blob[at + 16:at + 16 + n]))
        at += 16 + (n + 7) // 8 * 8
    return out


def _appended(engine, sid, k, n_feat):
    """the rows step k (just run) appended to the session's decode window: the window of parity (k & 1) ^ 1, last n_feat rows"""
    dw = [np.frombuffer(p, np.float32) for t, p in _sections(engine.session_snapshot(sid)) if t == 'DWF0']
    assert len(dw) == 2
    return dw[(k & 1) ^ 1][-n_feat:].copy()


def _rows(engine, sid, chunks, n_feat, before=None):
    """(outputs, appended decode-window rows of every step) of blocking pushes"""
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    outs, rows = [], []
    for k, c in enumerate(chunks):
        if before:
            before(k)
        outs.append(engine.session_push(sid, c, buf).copy())
        rows.append(_appended(engine, sid, k, n_feat))
    return outs, np.concatenate(rows)


def _pitched(engine, made, voice=0, **settings):
    sid = made.create(voice=voice)
    engine.session_pitch_correct(sid)
    engine.session_set_pitch_correct(sid, **(settings or SETTINGS))
    return sid


def _whole(engine, f0, **settings):
    s = dict(SETTINGS, **settings)
    return engine.pitch_correct(np.asarray(f0, np.float64), FS, HOP, s['key'], s['scale'], s['a4_hz'], s['retune_ms'], s['amount'])


# ---- 1 ------------------------------------------------------------------------------------------------------------------------
def _contours():
    rng = np.random.default_rng(11)
    t = np.arange(400) * HOP / 1000
    long = 55.0 + np.cumsum(rng.normal(0, 0.06, 60000))
    for a in rng.integers(0, 59900, 300):
        long[a:a + rng.integers(2, 60)] = np.nan
    return {'vibrato': 64.0 + 0.6 * np.sin(2 * np.pi * 5.5 * t), 'glide': np.linspace(57.0, 69.0, 900),
            'between': np.full(300, 64.5) + 0.04 * np.sin(np.arange(300) / 3.0), 'long gappy': long, 'silence': np.full(200, np.nan)}


def test_the_whole_signal_call_is_the_oracle(engine):
    cases, reported = 0, []
    for name, semis in _contours().items():
        f0 = np.where(np.isnan(semis), 0.0, 440.0 * 2.0 ** ((semis - 69.0) / 12.0))
        for key, scale, a4, retune, amount in ((0, 0xfff, 440.0, 0.0, 1.0), (2, MAJOR, 442.0, 30.0, 1.0),
                                               (9, PITCH_SCALES['minor'], 432.0, 250.0, 0.6),
                                               (5, 0b000010010001, 480.0, 1000.0, 1.0), (0, MAJOR, 400.0, 50.0, 0.0)):
            got = engine.pitch_correct(f0, FS, HOP, key, scale, a4, retune, amount)
            assert np.array_equal(got, engine.pitch_correct(f0, FS, HOP, key, scale, a4, retune, amount)), 'not repeatable'
            notes = []
            want = P.pitch_correct(f0, HOP, key, scale, a4, retune, amount, notes=notes)
            assert np.array_equal(got == 0, f0 == 0)
            if amount == 0:
                assert np.array_equal(got.view(np.int64), f0.view(np.int64))
            rel = np.abs(got - want) / np.where(want == 0, 1.0, np.abs(want))
            bad = np.flatnonzero(rel > 1e-12)
            if len(bad):
                # only a note choice can move a frame this far: the first such frame must sit at a decision boundary
                i = int(bad[0])
                j = [k for k, (fi, _, _) in enumerate(notes) if fi == i][0]
                n_prev = notes[j - 1][1] if j else P.NO_NOTE
                dist = P.boundary_distance(notes[j][2], key, scale, n_prev)
                reported.append((name, key, scale, i, notes[j][2], dist))
                assert dist < 1e-9, (name, key, scale, i, float(rel[i]))
                rel = rel[:i]
            cases += 1
            print(f'{name} key {key} scale {scale:#05x} retune {retune}: {len(f0)} frames, largest relative difference '
                  f'{float(rel.max()) if len(rel) else 0.0:.1e}')
    print(f'{cases} cases; frames at a decision boundary (name, key, scale, frame, s, distance): {reported}')


# ---- 2 ------------------------------------------------------------------------------------------------------------------------
def test_amount_zero_is_a_session_without_the_stage(engine, made):
    chunks = _speech(12, stream=1201)
    plain = _push(engine, made.create(), chunks)
    off = made.create()
    engine.session_pitch_correct(off)
    assert engine.session_get_pitch_correct(off) == dict(key=0, scale=0xfff, a4_hz=440.0, retune_ms=50.0, amount=0.0)
    assert _same(_push(engine, off, chunks), plain)
    on = made.create()
    engine.session_pitch_correct(on)
    engine.session_set_pitch_correct(on, **dict(SETTINGS, amount=0.0))
    assert _same(_push(engine, on, chunks), plain)
    voiced, mean, mx = engine.session_pitch_stats(on)
    assert voiced > 0 and mean == 0.0 and mx == 0.0


def _launch_windows(out_dir):
    """Child process of the launch-count test: returns (kernels the profiler saw, change of engine.launch_count) over 12 steps of a plain
    session, of one with the stage and of a plain one after it."""
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    _load(engine, synthetic.write_synthetic_models(out_dir / 'models', seed=0))
    engine.set_precision('fp16')
    chunks = _speech(12, stream=1211)
    counts = {}
    for name in ('plain', 'pitch', 'plain_after'):
        sid = engine.session_create(_cfg())
        if name == 'pitch':
            engine.session_pitch_correct(sid)
            engine.session_set_pitch_correct(sid, **SETTINGS)
        counts[name] = _window(engine, out_dir, lambda: _push(engine, sid, chunks))
        engine.session_destroy(sid)
    return counts


def test_one_kernel_per_step_and_none_for_other_sessions(tmp_path):
    counts = _run_child(tmp_path, 'test_gpu_pitch', '_launch_windows')
    for name, (seen, counted) in counts.items():
        print(f'{name}: {counted} kernels counted over 12 steps, {seen} seen by the profiler')
        assert seen == counted, name
    assert counts['pitch'][1] - counts['plain'][1] == 1 * 12
    assert counts['plain_after'][1] == counts['plain'][1]


# ---- 3 ------------------------------------------------------------------------------------------------------------------------
def _stable_cents(engine, y, fs=FS):
    """cents from the nearest chromatic note (A4 = 442) of the voiced frames of ryk_world_analyze(y) whose f0 moves less than 10 cents
    against both neighbours (WORLD places pulses on whole samples, so a synthesized steady tone re-analyses with a few cents of jitter)"""
    a = engine.world_analyze(np.asarray(y, np.float64), fs, HOP, 71.0, 800.0, 1024, 8, 0.466)
    f0 = np.asarray(a['f0'], np.float64)
    v = f0 > 0
    s = np.full(len(f0), np.nan)
    s[v] = 69 + 12 * np.log2(f0[v] / 442.0)
    steady = v[1:-1] & v[:-2] & v[2:] & (np.abs(s[1:-1] - s[:-2]) < 0.1) & (np.abs(s[1:-1] - s[2:]) < 0.1)
    mid = s[1:-1][steady]
    return np.abs(mid - np.round(mid)) * 100


@pytest.mark.parametrize('extras', [EXTRA, (0.025, 0.1, 0.025)])
def test_the_session_gives_its_synthesizer_the_whole_signal_correction(engine, made, extras):
    steps = 14
    chunks = _speech(steps, stream=1221)
    cfg = _cfg()
    cfg.encode_extra_time, cfg.convert_extra_time, cfg.decode_extra_time = extras
    n_feat = round(T * 1000 / HOP)
    sids = []
    try:
        plain = engine.session_create(cfg)
        sids.append(plain)
        _, rows_plain = _rows(engine, plain, chunks, n_feat)
        hard = dict(SETTINGS, scale='chromatic', retune_ms=0.0)
        for settings in (SETTINGS, hard):
            sid = engine.session_create(cfg)
            sids.append(sid)
            engine.session_pitch_correct(sid)
            engine.session_set_pitch_correct(sid, **settings)
            _, rows = _rows(engine, sid, chunks, n_feat)
            want = _whole(engine, rows_plain.astype(np.float64), **settings).astype(np.float32)
            assert (rows_plain > 0).sum() > 100
            assert np.array_equal(rows.view(np.uint32), want.view(np.uint32)), (extras, settings)
            assert not np.array_equal(rows, rows_plain)
    finally:
        for sid in sids:
            engine.session_destroy(sid)


def test_the_output_sits_on_scale_notes(engine, made):
    """A sustained sung note (a steady harmonic tone) through a session with a hard chromatic snap: the output re-analysed with
    ryk_world_analyze sits on notes of A4 = 442 Hz.  Tolerance: the median steady voiced frame within 5 cents of a note and 90 % within
    15 cents -- the synthesizer is given frames exactly on a note, and WORLD's re-analysis of a synthesized steady tone is accurate to a
    few cents."""
    chunks = _tone(14, hz=150.0)
    y0 = np.concatenate(_push(engine, made.create(), chunks))
    y = np.concatenate(_push(engine, _pitched(engine, made, **dict(SETTINGS, scale='chromatic', retune_ms=0.0)), chunks))
    cents, cents0 = _stable_cents(engine, y), _stable_cents(engine, y0)
    print(f'output re-analysed: {len(cents)} steady voiced frames, median {np.median(cents):.2f} cents from a note, 90th percentile '
          f'{np.percentile(cents, 90):.2f} (without the stage: {len(cents0)} frames, median {np.median(cents0):.2f})')
    assert len(cents) >= 100 and np.median(cents) <= 5.0 and np.percentile(cents, 90) <= 15.0


# ---- 4 ------------------------------------------------------------------------------------------------------------------------
def test_a_setting_change_lands_on_the_next_submitted_step(engine, made):
    steps, j1 = 10, 4
    chunks = _speech(steps, stream=1231)
    s1 = dict(key='A', scale='minor', a4_hz=440.0, retune_ms=0.0, amount=0.8)
    piped = _pitched(engine, made)
    buf = np.empty(engine.session_io_geometry(piped)['max_out'])
    tickets, got = [], []
    for k, c in enumerate(chunks):                 # five submitted before the first collect: the change is made with chunks in flight
        if k == j1:
            engine.session_set_pitch_correct(piped, **s1)
            assert engine.session_get_pitch_correct(piped)['key'] == 9
        tickets.append(engine.session_submit(piped, c))
        if k == 4:
            got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
            tickets = []
    got += [engine.session_collect(piped, t, buf).copy() for t in tickets]
    blocking = _pitched(engine, made)
    want = _push(engine, blocking, chunks, before=lambda k: k == j1 and engine.session_set_pitch_correct(blocking, **s1))
    assert _same(got, want)
    assert not _same(got, _push(engine, _pitched(engine, made), chunks))


# ---- 5 ------------------------------------------------------------------------------------------------------------------------
def test_group_members_and_voice_switches_keep_the_correction(engine, made, full_models, second_voice_files):
    steps, switch_at = 8, 4
    chunks = _speech(steps, stream=1241)
    engine.set_precision('fp32')
    alone = _push(engine, _pitched(engine, made), chunks)
    a, b = _pitched(engine, made), _pitched(engine, made, key=3, scale='minor', retune_ms=0.0, amount=0.5)
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
    n_feat = round(T * 1000 / HOP)
    reference = made.create(voice=v1)
    _, rows_plain = _rows(engine, reference, chunks, n_feat, before=lambda k: k == switch_at and engine.session_set_voice(reference, v2))
    switched = _pitched(engine, made, voice=v1)
    _, rows = _rows(engine, switched, chunks, n_feat, before=lambda k: k == switch_at and engine.session_set_voice(switched, v2))
    want = _whole(engine, rows_plain.astype(np.float64)).astype(np.float32)
    assert np.array_equal(rows.view(np.uint32), want.view(np.uint32))


# ---- 6 ------------------------------------------------------------------------------------------------------------------------
def test_snapshot_and_restore_continue_bitwise(engine, made):
    steps, cut = 12, 5
    chunks = _speech(steps, stream=1251)
    whole = _push(engine, _pitched(engine, made), chunks)
    a = _pitched(engine, made)
    first = _push(engine, a, chunks[:cut])
    engine.session_set_pitch_correct(a, retune_ms=120.0)         # a setting not yet submitted travels too
    blob = engine.session_snapshot(a)
    b = engine.session_restore(blob)
    made.sids.append(b)
    assert engine.session_get_pitch_correct(b) == engine.session_get_pitch_correct(a)
    d = describe_snapshot(blob)
    assert d['pitch_correct'] == engine.session_get_pitch_correct(a)
    rest_a = _push(engine, a, chunks[cut:])
    rest_b = _push(engine, b, chunks[cut:])
    assert _same(rest_a, rest_b)
    # without the setting change the continued stream is the uninterrupted one
    c = _pitched(engine, made)
    head = _push(engine, c, chunks[:cut])
    d2 = engine.session_restore(engine.session_snapshot(c))
    made.sids.append(d2)
    assert _same(head + _push(engine, d2, chunks[cut:]), whole)
    assert _same(first, whole[:cut])
    # a session without the stage writes the sections it wrote before: the pitched blob's without PTCH, PTCP and PTCS
    plain = made.create()
    _push(engine, plain, chunks[:cut])
    tags = [t for t, _ in describe_snapshot(engine.session_snapshot(plain))['sections']]
    pitched = [t for t, _ in d['sections']]
    assert not {'PTCH', 'PTCP', 'PTCS'} & set(tags) and describe_snapshot(engine.session_snapshot(plain))['pitch_correct'] is None
    assert [t for t in pitched if t not in ('PTCH', 'PTCP', 'PTCS')] == tags
    assert pitched.count('PTCH') == pitched.count('PTCP') == pitched.count('PTCS') == 1


# ---- 7 ------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_cycles_return_memory(engine, made):
    import torch
    chunks = _speech(5, stream=1261)
    sid, twin, plain = _pitched(engine, made), _pitched(engine, made), made.create()

    def refused(call):
        before = engine.launch_count
        with pytest.raises(RykError) as err:
            call()
        assert str(err.value)
        assert engine.launch_count == before
    f0 = np.full(100, 220.0)
    bad = [dict(key=12), dict(key=-1), dict(scale=0), dict(scale=0x1000), dict(a4_hz=399.0), dict(a4_hz=math.nan), dict(a4_hz=481.0),
           dict(retune_ms=-1.0), dict(retune_ms=1001.0), dict(retune_ms=math.inf), dict(amount=1.01), dict(amount=-0.1),
           dict(amount=math.nan)]
    for b in bad:
        s = dict(SETTINGS, **b)
        refused(lambda: engine.pitch_correct(f0, FS, HOP, s['key'], s['scale'], s['a4_hz'], s['retune_ms'], s['amount']))
    refused(lambda: engine.pitch_correct(f0, 0, HOP))
    refused(lambda: engine.pitch_correct(f0, FS, 0.0))
    for call in (lambda: engine.session_set_pitch_correct(plain, **SETTINGS), lambda: engine.session_get_pitch_correct(plain),
                 lambda: engine.session_pitch_stats(plain), lambda: engine.session_pitch_correct(99999),
                 lambda: engine.session_get_pitch_correct(99999)):
        refused(call)
    outs = _push(engine, sid, chunks[:2])
    refused(lambda: engine.session_pitch_correct(sid))                  # ran a step
    refused(lambda: engine.session_pitch_correct(twin))                 # enabled twice
    before = engine.session_get_pitch_correct(sid)
    for b in bad:
        refused(lambda: engine.session_set_pitch_correct(sid, **b))
    assert engine.session_get_pitch_correct(sid) == before
    outs += _push(engine, sid, chunks[2:])
    assert _same(outs, _push(engine, twin, chunks))
    free = {}
    for cycle in range(1, 13):
        s = engine.session_create(_cfg())
        engine.session_pitch_correct(s)
        engine.session_set_pitch_correct(s, **SETTINGS)
        engine.session_push(s, chunks[0])
        engine.session_push(s, chunks[1])
        engine.session_destroy(s)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 session cycles with pitch correction')
    assert abs(grown) < 4.0


# ---- 8 ------------------------------------------------------------------------------------------------------------------------
def test_run_autotune_is_the_pipelines_correction(engine, small_models, tmp_path):
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
    x, rate = wave_io.read_wav(Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav')
    wave_io.write_wav(tmp_path / 'in.wav', np.asarray(x, np.float32), FS)
    run_mod.main(['--config_path', str(tmp_path / 'config.yaml'), '--wav_in', str(tmp_path / 'in.wav'), '--wav_out',
                  str(tmp_path / 'tuned.wav'), '--autotune', 'F#:minor', '--retune_ms', '20', '--autotune_amount', '0.9'])
    config = Config.from_yaml(tmp_path / 'config.yaml')
    param = YukarinConverter.make_yukarin_converter(**paths).acoustic_converter.config.dataset.acoustic_param
    wave = wave_io.load_wave(tmp_path / 'in.wav', config.input_rate, engine=engine).wave

    def pipeline_run(**kw):
        pipe = RealtimePipeline(config, acoustic_param=param, engine=engine, **kw)
        got = []
        try:
            for i in range(len(wave) // config.in_audio_chunk):
                got.append(pipe.process(wave[i * config.in_audio_chunk:(i + 1) * config.in_audio_chunk]))
            got.extend(pipe.drain())
            pipe.flush()
            stats = pipe.pitch_stats() if kw else None
        finally:
            pipe.close()
        return np.concatenate(got), stats

    def played(w):
        """the output chunks that carry sound: where the loop plays silence because nothing was ready yet depends on timing"""
        w = np.asarray(w)
        frames = w[:len(w) // config.out_audio_chunk * config.out_audio_chunk].reshape(-1, config.out_audio_chunk)
        return frames[np.any(frames != 0, axis=1)]

    mine, stats = pipeline_run(pitch_correct=dict(key='F#', scale='minor', retune_ms=20.0, amount=0.9))
    plain, _ = pipeline_run()
    ran = wave_io.load_wave(tmp_path / 'tuned.wav', FS, engine=engine).wave
    assert len(played(mine)) >= 10 and np.array_equal(played(ran), played(mine))
    assert not np.array_equal(played(plain), played(mine))
    print(f'run.py --autotune F#:minor --retune_ms 20 --autotune_amount 0.9: last chunk {stats[0]} voiced frames, mean {stats[1]:.1f} '
          f'cents, largest {stats[2]:.1f} cents')
