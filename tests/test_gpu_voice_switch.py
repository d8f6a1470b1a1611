"""Switching a running session to another voice between steps (ryk_session_set_voice), keeping its stream state.

  * the switched stream is the oracle's stream with stage1 / stage2 / f0_stats swapped between pushes (A -> B at k, B -> A at k2), FP16
    base 64 and FP32 base 16, and differs from both single-voice streams after k;
  * the steps before a switch are bitwise an unswitched session's; a same-voice switch is bitwise no call; an FP32 session switched in
    a group is bitwise the same session switched alone; in a mixed group the members that do not switch are bitwise a run without it;
  * the call launches nothing and the steps after it launch what a session created on the new voice launches, allocating nothing;
  * the f0 map becomes the new voice's, a map set after the switch lands on the next step, the measurement and the formant carry over,
    follow mode keeps its measured input side;
  * device rates with a re-blocker, and RealtimePipeline.set_voice, switch mid-stream;
  * refusals change nothing; the voices' locks move; switch cycles return their memory.

The voices are loaded on the shared engine from their own seeded model files and destroyed at the end.
"""
import functools
import math

import numpy as np
import pytest
import scipy.signal as ss

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import RykError, SessionConfig

from .formant_oracle import FormantStreamOracle

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()
FS = 24000
EXTRA = (0.0, 0.5, 0.0)
TOL = 1e-3                      # sample RMSE of the FP16 and FP32 session tests (tests/test_gpu_parity.py, test_gpu_voices.py)
SEMITONE = math.log(2.0) / 12.0


def _cfg(T=0.3):
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                         encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                         vocoder_buffer_size=1024)


def _chunks(steps, stream, T=0.3):
    n = round(T * FS)
    x = synthetic.synthetic_speech((steps + 1) * T, stream=stream)
    return [np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32) for k in range(steps)]


def _rmse(a, b):
    a, b = np.concatenate(a), np.concatenate(b)
    assert len(a) == len(b)
    return float(np.sqrt(np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)))


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _load_voice(engine, paths):
    from realtime_yukarin_b200.models import load_voice
    v = engine.voice_create()
    load_voice(engine, v, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                     'target_statistics_path')})
    return v


@pytest.fixture(scope='module')
def voice_files(tmp_path_factory):
    """Three base-64 voices (seeds 51..53) and two base-16 ones (seeds 54, 55), none shared with the other test modules."""
    out = {seed: synthetic.write_synthetic_models(tmp_path_factory.mktemp(f'switch{seed}'), seed=seed) for seed in (51, 52, 53)}
    for seed in (54, 55):
        out[seed] = synthetic.write_synthetic_models(tmp_path_factory.mktemp(f'switch{seed}'), seed=seed, base1=16, base2=16)
    return out


@pytest.fixture(scope='module')
def voices(engine, voice_files):
    """{'A', 'B', 'C'} base 64 and {'a', 'b'} base 16 -> (voice id, model files), loaded on the shared engine; destroyed afterwards."""
    engine.set_precision('fp16')
    ids = {name: (_load_voice(engine, voice_files[seed]), voice_files[seed])
           for name, seed in (('A', 51), ('B', 52), ('C', 53), ('a', 54), ('b', 55))}
    yield ids
    for v, _ in ids.values():
        engine.voice_destroy(v)


class _Made:
    """Sessions, groups, re-blockers and voices of a test, destroyed whatever failed; the engine's modes restored."""

    def __init__(self, engine):
        self.engine, self.sids, self.gids, self.voices = engine, [], [], []

    def session(self, voice, T=0.3):
        self.sids.append(self.engine.session_create(_cfg(T), voice=voice))
        return self.sids[-1]

    def group(self, sids):
        self.gids.append(self.engine.group_create(sids))
        return self.gids[-1]

    def close(self):
        e = self.engine
        e.set_precision('fp16')
        e.set_stage1_fused(True)
        for items, destroy in ((self.gids, e.group_destroy), (self.sids, e.session_destroy), (self.voices, e.voice_destroy)):
            while items:
                destroy(items.pop())


@pytest.fixture
def made(engine, voices):
    engine.set_precision('fp16')
    m = _Made(engine)
    yield m
    m.close()


def _run(engine, sid, chunks, switch=None, depth=3, before=None):
    """submit / collect with up to `depth` chunks in flight.  In front of step k in `switch` (k -> voice id) every chunk in flight is
    collected and the session switched; before(k) runs after that, in front of the submit of step k."""
    switch = switch or {}
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    tickets, outs = [], []

    def collect():
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    for k, c in enumerate(chunks):
        if k in switch:
            while tickets:
                collect()
            engine.session_set_voice(sid, switch[k])
        if before:
            before(k)
        tickets.append(engine.session_submit(sid, c))
        if len(tickets) > depth:
            collect()
    while tickets:
        collect()
    return outs


def _run_group(engine, gid, chunks_of, steps, switch=None, depth=3):
    """group_submit / _collect with up to `depth` steps in flight; chunks_of[sid][k] is the chunk of member sid at step k.  In front of
    step k in `switch` (k -> (sid, voice id)) every step in flight is collected and the member switched.  Returns {sid: outputs}."""
    switch = switch or {}
    members = engine.group_members(gid)
    cap = max(engine.session_io_geometry(s)['max_out'] for s in members)
    bufs = [[np.empty(cap) for _ in members] for _ in range(8)]
    outs = {s: [] for s in members}
    tickets = []

    def collect():
        t = tickets.pop(0)
        for s, o in zip(members, engine.group_collect(gid, t, bufs[t % 8])):
            outs[s].append(o.copy())
    for k in range(steps):
        if k in switch:
            while tickets:
                collect()
            engine.session_set_voice(*switch[k])
            assert engine.group_members(gid) == members              # a member's slot does not move
        tickets.append(engine.group_submit(gid, [chunks_of[s][k] for s in members]))
        if len(tickets) > depth:
            collect()
    while tickets:
        collect()
    return outs


@functools.lru_cache(maxsize=None)
def _npz(path):
    return onets.load_npz(path)


def _oracle_voice(paths):
    from realtime_yukarin_b200.models import F0Converter
    return (_npz(str(paths['stage1_model_path'])), _npz(str(paths['stage2_model_path'])),
            F0Converter(paths['input_statistics_path'], paths['target_statistics_path']).stats())


def _oracle(paths_at, chunks, T=0.3, stats_at=None, formant=1.0):
    """The oracle's stream with the nets and f0 statistics of the voice whose model files are paths_at(k) swapped in front of push k;
    stats_at(k), when given, replaces the f0 statistics."""
    p1, p2, stats = _oracle_voice(paths_at(0))
    orc = FormantStreamOracle(CFG, p1, p2, stats, buffer_time=T, extra=EXTRA, backend='torch')
    orc.formant_ratio = formant
    outs = []
    for k, c in enumerate(chunks):
        orc.stage1, orc.stage2, orc.f0_stats = _oracle_voice(paths_at(k))
        if stats_at:
            orc.f0_stats = stats_at(k)
        outs.append(orc.push(c))
    return outs


def _refused(engine, call, needle):
    before = engine.launch_count
    with pytest.raises(RykError, match=needle):
        call()
    assert engine.launch_count == before


# ---- 1, 2: against the oracle; the steps before the switch ----------------------------------------------------------------------
@pytest.mark.parametrize('T,steps,k,k2', [(0.3, 9, 3, 6), (1.0, 4, 1, 3)])
def test_fp16_switch_is_the_switching_oracle(engine, voices, made, T, steps, k, k2):
    (va, fa), (vb, fb) = voices['A'], voices['B']
    chunks = _chunks(steps, stream=701, T=T)
    sid, plain = made.session(va, T), made.session(va, T)
    outs = _run(engine, sid, chunks, {k: vb, k2: va})
    assert engine.session_voice(sid) == va
    unswitched = _run(engine, plain, chunks)
    assert _same(outs[:k], unswitched[:k])
    refs = _oracle(lambda j: fb if k <= j < k2 else fa, chunks, T)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    err = _rmse(outs, refs)
    only_a, only_b = _oracle(lambda j: fa, chunks[:k2], T), _oracle(lambda j: fb, chunks[:k2], T)
    apart_a, apart_b = _rmse(outs[k:k2], only_a[k:k2]), _rmse(outs[k:k2], only_b[k:k2])
    print(f'T={T}: A -> B at {k}, B -> A at {k2}: sample RMSE {err:.3e} to the switching oracle; steps {k}..{k2 - 1} differ from the '
          f'A-only oracle by {apart_a:.3e}, from the B-only oracle by {apart_b:.3e}')
    assert err <= TOL
    # After the switch the rows handed to the synthesizer are the B-only session's, so the B-only stream differs only by the
    # synthesizer's history (pulse phase, overlap-add carry): about 1e-3 at 0.3 s and 6e-4 at 1.0 s on these voices, still more than
    # 100 times the distance to the switching oracle.  The A-only stream differs by the voices' own distance.
    assert apart_a > max(100 * err, TOL) and apart_b > 100 * err


def test_fp32_switch_alone_and_grouped(engine, voices, made):
    """FP32, base 16: the oracle's bound of the FP32 session tests (a stream RMSE of 1e-3 leaves room for DESIGN.md §5 lesson 2, a
    pulse placed one sample off); a session switched as the one member of a group (several voices need FP16) is bitwise it alone."""
    (va, fa), (vb, fb) = voices['a'], voices['b']
    steps, k, k2 = 9, 3, 6
    chunks = _chunks(steps, stream=711)
    engine.set_precision('fp32')
    alone, grouped, plain = made.session(va), made.session(va), made.session(va)
    gid = made.group([grouped])
    out_alone = _run(engine, alone, chunks, {k: vb, k2: va})
    out_group = _run_group(engine, gid, {grouped: chunks}, steps, {k: (grouped, vb), k2: (grouped, va)})[grouped]
    unswitched = _run(engine, plain, chunks)
    assert _same(out_alone, out_group)
    assert _same(out_alone[:k], unswitched[:k])
    refs = _oracle(lambda j: fb if k <= j < k2 else fa, chunks)
    err = _rmse(out_alone, refs)
    apart = _rmse(out_alone[k:k2], unswitched[k:k2])
    print(f'FP32 base 16: sample RMSE {err:.3e} to the switching oracle; steps {k}..{k2 - 1} moved by {apart:.3e}')
    assert err <= TOL
    assert apart > max(100 * err, TOL)


def test_same_voice_is_no_call(engine, voices, made):
    va = voices['A'][0]
    steps, k = 7, 3
    chunks = _chunks(steps, stream=721)
    a, b = made.session(va), made.session(va)
    before = engine.launch_count

    def same(j):
        if j == k:          # with chunks in flight: a no-op does not wait for them
            engine.session_set_voice(a, va)
    out_a = _run(engine, a, chunks, before=same)
    count_a = engine.launch_count - before
    before = engine.launch_count
    out_b = _run(engine, b, chunks)
    assert _same(out_a, out_b)
    assert count_a == engine.launch_count - before


def test_mixed_group_members_that_do_not_switch_are_unchanged(engine, voices, made):
    (va, fa), (vb, fb), (vc, fc) = voices['A'], voices['B'], voices['C']
    steps, k, k2 = 8, 3, 6
    pattern = (va, vb, va, vc)
    xs = [_chunks(steps, stream=730 + i) for i in range(len(pattern))]

    def run(switch):
        sids = [made.session(v) for v in pattern]
        gid = made.group(sids)
        outs = _run_group(engine, gid, dict(zip(sids, xs)), steps,
                          {k: (sids[0], vc), k2: (sids[0], vb)} if switch else None)
        if switch:
            assert engine.session_voice(sids[0]) == vb
        return [outs[s] for s in sids]
    switched, untouched = run(True), run(False)
    for i in range(1, len(pattern)):
        assert _same(switched[i], untouched[i]), i
    assert _same(switched[0][:k], untouched[0][:k])
    alone = _run(engine, made.session(va), xs[0], {k: vc, k2: vb})
    err = _rmse(switched[0], alone)
    print(f'switched member vs the same switches alone: sample RMSE {err:.3e}')
    assert err <= 1e-4
    assert _rmse(switched[0][k:], untouched[0][k:]) > max(100 * err, TOL)


# ---- 3: launches and allocations ------------------------------------------------------------------------------------------------
def test_the_call_launches_nothing_and_later_steps_are_a_new_sessions(engine, voices, made):
    import torch
    va, vb = voices['A'][0], voices['B'][0]
    steps, k = 10, 4
    chunks = _chunks(steps, stream=741)
    sid, fresh = made.session(va), made.session(vb)
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])

    def per_step(s, j0=0, switch_at=None):
        counts, free = [], {}
        for j in range(j0, steps):
            if j == switch_at:
                before = engine.launch_count
                engine.session_set_voice(s, vb)
                assert engine.launch_count == before
            before = engine.launch_count
            engine.session_push(s, chunks[j], buf)
            counts.append(engine.launch_count - before)
            free[j] = torch.cuda.mem_get_info()[0]
        return counts, free
    switched, free = per_step(sid, switch_at=k)
    created, _ = per_step(fresh)
    print(f'kernels per step: switched {switched}, created on the new voice {created}')
    assert switched[k:] == created[k:]
    grown = (free[k + 1] - free[steps - 1]) / 2**20
    print(f'device memory taken by steps {k + 2}..{steps - 1}: {grown:.2f} MiB')
    assert abs(grown) < 1.0                                          # no step after the first two allocates


# ---- 4: the f0 map, the measurement, follow mode and the formant ratio ----------------------------------------------------------
def test_f0_map_becomes_the_new_voices(engine, voices, made):
    (va, fa), (vb, fb) = voices['A'], voices['B']
    steps, k = 7, 3
    chunks = _chunks(steps, stream=751)
    sid, shifted, fresh = made.session(va), made.session(va), made.session(vb)
    engine.session_set_f0_map(sid, semitones=3)                      # a caller's offset does not survive the switch
    _run(engine, sid, chunks[:k])
    engine.session_set_voice(sid, vb)
    assert engine.session_get_f0_map(sid) == engine.session_get_f0_map(fresh)
    # a map set between the switch and the next submit lands on that step
    stats_b = _oracle_voice(fb)[2]
    up = (stats_b[0], stats_b[1], stats_b[2] + 12 * SEMITONE, stats_b[3])
    outs = _run(engine, shifted, chunks, {k: vb}, before=lambda j: j == k and engine.session_set_f0_map(shifted, semitones=12))
    refs = _oracle(lambda j: fb if j >= k else fa, chunks, stats_at=lambda j: up if j >= k else _oracle_voice(fa)[2])
    plain = _run(engine, made.session(va), chunks, {k: vb})
    err, moved = _rmse(outs, refs), _rmse(outs[k:], plain[k:])
    print(f'+12 semitones set after the switch: sample RMSE {err:.3e} to the oracle, {moved:.3e} from the switch without it')
    assert err <= TOL
    assert moved > 10 * TOL


def test_measurement_and_follow_mode_carry_over(engine, voices, made):
    va, vb = voices['A'][0], voices['B'][0]
    steps, k, min_voiced, floor = 9, 4, 60, 0.05
    chunks = _chunks(steps, stream=761)
    measured, unswitched = made.session(va), made.session(va)
    for s in (measured, unswitched):
        engine.session_f0_measure(s)
    _run(engine, measured, chunks, {k: vb})
    _run(engine, unswitched, chunks)
    assert engine.session_f0_measured(measured) == engine.session_f0_measured(unswitched)
    # follow mode is bitwise a host that switches and then sets the measured input side before every step
    ahead, following, by_hand = made.session(va), made.session(va), made.session(va)
    engine.session_f0_measure(ahead)
    engine.session_f0_measure(following)
    engine.session_f0_follow(following, True, min_voiced_frames=min_voiced, sd_floor=floor)
    buf = np.empty(engine.session_io_geometry(ahead)['max_out'])
    reached = []

    def host_rule(j):
        engine.session_push(ahead, chunks[j], buf)
        n, mean, std = engine.session_f0_measured(ahead)               # includes the frames of chunk j
        if n >= min_voiced:
            reached.append(j)
            engine.session_set_f0_map(by_hand, in_mean=mean, in_std=max(std, floor))
    out_hand = _run(engine, by_hand, chunks, {k: vb}, depth=0, before=host_rule)
    out_follow = _run(engine, following, chunks, {k: vb})
    assert reached and reached[0] < k
    assert _same(out_follow, out_hand)
    plain = _run(engine, made.session(va), chunks, {k: vb})
    assert not _same(out_follow[k:], plain[k:])


def test_formant_ratio_carries_over(engine, voices, made):
    (va, fa), (vb, fb) = voices['A'], voices['B']
    steps, k, ratio = 7, 3, 1.25
    chunks = _chunks(steps, stream=771)
    sid = made.session(va)
    engine.session_set_formant(sid, ratio=ratio)
    outs = _run(engine, sid, chunks, {k: vb})
    assert engine.session_get_formant(sid) == ratio
    refs = _oracle(lambda j: fb if j >= k else fa, chunks, formant=ratio)
    err = _rmse(outs, refs)
    print(f'formant ratio {ratio} through the switch: sample RMSE {err:.3e} to the oracle')
    assert err <= TOL


# ---- 5, 8: device rates with a re-blocker, RealtimePipeline.set_voice -----------------------------------------------------------
def _ratio(r_from, r_to):
    g = math.gcd(r_from, r_to)
    return r_to // g, r_from // g


@pytest.mark.parametrize('rate', [24000, 48000])
def test_pipeline_and_device_rates_switch_mid_stream(engine, voices, made, rate):
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import Item, OutputReblocker, RealtimePipeline
    (va, fa), (vb, fb) = voices['A'], voices['B']
    K, k, k2, T = 9, 3, 6, 0.3
    switch = {k: vb, k2: va}
    x = wave_io.resample(synthetic.synthetic_speech(K * T + 0.2, stream=781), FS, rate, engine) if rate != FS else \
        synthetic.synthetic_speech(K * T + 0.2, stream=781)
    fields = dict(input_device_name=None, output_device_name=None, input_rate=rate, output_rate=rate, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2])
    cfg = Config(extract_f0_mode=VocodeMode.WORLD, **fields, **{p: fa[p] for p in (
        'input_statistics_path', 'target_statistics_path', 'stage1_model_path', 'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})
    n_in = cfg.in_audio_chunk
    chunks = [np.ascontiguousarray(x[j * n_in:(j + 1) * n_in], np.float32) for j in range(K)]
    pipe = RealtimePipeline(cfg, engine=engine, depth=3, voice=va)
    try:
        for j, c in enumerate(chunks):
            if j in switch:
                pipe.set_voice(switch[j])
            pipe.put(Item(item=c, index=j))
        got = [pipe.get() for _ in range(K)]
    finally:
        pipe.close()
    assert [it.index for it in got] == list(range(K))
    # the engine-level stream at the models' rate, switched at the same chunks
    n = round(T * FS)
    if rate != FS:
        _, _, D = wave_io.stream_input_geometry(rate, FS, T)
        up, down = _ratio(rate, FS)
        xm = np.concatenate([np.zeros(D, np.float32), engine.resample_poly(x, up, down, wave_io.resample_filter(up, down))])
    else:
        xm = x
    native = _run(engine, made.session(va), [np.ascontiguousarray(xm[j * n:(j + 1) * n], np.float32) for j in range(K)], switch)
    if rate != FS:
        up, down = _ratio(FS, rate)
        z = ss.resample_poly(np.concatenate(native), up, down, window=wave_io.resample_filter(up, down) / up)
        M = [wave_io.stream_output_count(int(c), rate, FS) for c in np.cumsum([len(v) for v in native])]
        # the switched session at the device rates returns resample_poly of the switched model-rate stream
        sid = made.session(va)
        engine.session_set_input_rate(sid, rate)
        engine.session_set_output_rate(sid, rate)
        dev = _run(engine, sid, chunks, switch)
        peak = np.abs(np.concatenate(native)).max()
        assert [len(o) for o in dev] == list(np.diff([0] + M))
        assert np.abs(np.concatenate(dev) - z[:M[-1]]).max() <= 1e-12 * peak
        pieces = [z[(M[j - 1] if j else 0):M[j]] for j in range(K)]
    else:
        pieces = native
    rb = OutputReblocker(cfg.out_audio_chunk, cfg.output_silent_threshold, max_in=max(len(p) for p in pieces) + 1, engine=engine)
    played = 0
    try:
        for j, it in enumerate(got):
            ref = rb.push(pieces[j])
            assert (it.item is None) == (ref is None), j
            if ref is not None:
                played += 1
                assert np.abs(it.item - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), j
    finally:
        rb.close()
    assert played > 0


# ---- 6: refusals ----------------------------------------------------------------------------------------------------------------
def _mismatched_voice(engine, made, narrow_files):
    """A voice with both models loaded whose stage-1 net takes 10 channels (order 9) instead of the session's 9."""
    from realtime_yukarin_b200.engine import _unet_layer_shapes
    from realtime_yukarin_b200.models import upload_unet
    v = engine.voice_create()
    made.voices.append(v)
    engine.model_create(1, 10, 10, 16, voice=v)
    for i, (tr, cin, cout, k) in enumerate(_unet_layer_shapes(1, 10, 10, 16)):
        W = np.zeros(((cin, cout) if tr else (cout, cin)) + (k,), np.float32)
        engine.model_set_layer(1, i, W, np.ones(cout, np.float32), np.zeros(cout, np.float32), voice=v)
    upload_unet(engine, 2, onets.load_npz(narrow_files['stage2_model_path']), voice=v)
    return v


def _voice_without_f0_stats(engine, made, files):
    from realtime_yukarin_b200.models import upload_unet
    v = engine.voice_create()
    made.voices.append(v)
    upload_unet(engine, 1, onets.load_npz(files['stage1_model_path']), voice=v)
    upload_unet(engine, 2, onets.load_npz(files['stage2_model_path']), voice=v)
    return v


def test_refusals_change_nothing(engine, voices, made):
    (va, fa), (vb, fb), (vc, fc), (vn, fn) = voices['A'], voices['B'], voices['C'], voices['a']
    steps = 7
    chunks = _chunks(steps, stream=791)
    s, twin = made.session(va), made.session(va)
    for x in (s, twin):
        engine.session_f0_measure(x)
        engine.session_f0_follow(x, True, min_voiced_frames=60)
    buf = np.empty(engine.session_io_geometry(s)['max_out'])
    outs = {x: [engine.session_push(x, c, buf).copy() for c in chunks[:2]] for x in (s, twin)}
    map_before = engine.session_get_f0_map(s)
    _refused(engine, lambda: engine.session_set_voice(10 ** 6, vb), 'no such session')
    _refused(engine, lambda: engine.session_set_voice(s, 10 ** 6), 'no such voice')
    empty = engine.voice_create()
    made.voices.append(empty)
    engine.model_create(1, 9, 9, 64, voice=empty)
    _refused(engine, lambda: engine.session_set_voice(s, empty), 'load')
    _refused(engine, lambda: engine.session_set_voice(s, _mismatched_voice(engine, made, fn)), 'order')
    _refused(engine, lambda: engine.session_set_voice(s, _voice_without_f0_stats(engine, made, fc)), 'follow mode')
    engine.set_precision('fp32')
    _refused(engine, lambda: engine.session_set_voice(s, vb), 'precision')
    engine.set_precision('fp16')
    engine.set_stage1_fused(False)
    _refused(engine, lambda: engine.session_set_voice(s, vb), 'stage-1 mode')
    engine.set_stage1_fused(True)
    for x in (s, twin):
        t = engine.session_submit(x, chunks[2])
        if x == s:
            _refused(engine, lambda: engine.session_set_voice(s, vb), 'collect')
        outs[x].append(engine.session_collect(x, t, buf).copy())
    assert engine.session_voice(s) == va and engine.session_get_f0_map(s) == map_before
    for x in (s, twin):
        outs[x] += [engine.session_push(x, c, buf).copy() for c in chunks[3:]]
    assert _same(outs[s], outs[twin])
    # a group refusal leaves the whole group as it was
    xs = [_chunks(steps, stream=795 + i) for i in range(2)]

    def group(refuse):
        sids = [made.session(va), made.session(vb)]
        gid = made.group(sids)
        got = _run_group(engine, gid, dict(zip(sids, xs)), 2)
        if refuse:
            _refused(engine, lambda: engine.session_set_voice(sids[0], vn), 'same')          # a base-16 stage 2 in a base-64 group
            t = engine.group_submit(gid, [x[2] for x in xs])
            _refused(engine, lambda: engine.session_set_voice(sids[0], vc), 'collect')
            bufs = [np.empty(engine.session_io_geometry(sids[0])['max_out']) for _ in sids]
            for s_, o in zip(sids, engine.group_collect(gid, t, bufs)):
                got[s_].append(o.copy())
            rest = _run_group(engine, gid, {s_: c[3:] for s_, c in zip(sids, xs)}, steps - 3)
        else:
            rest = _run_group(engine, gid, {s_: c[2:] for s_, c in zip(sids, xs)}, steps - 2)
        assert [engine.session_voice(x) for x in sids] == [va, vb]
        return [got[x] + rest[x] for x in sids]
    refused, plain = group(True), group(False)
    for i in range(2):
        assert _same(refused[i], plain[i]), i


# ---- 7: voice locks and memory ----------------------------------------------------------------------------------------------------
def test_voice_locks_move_and_cycles_return_memory(engine, voices, voice_files, made):
    import torch
    va, vb, vc = voices['A'][0], voices['B'][0], voices['C'][0]
    chunks = _chunks(3, stream=801)
    own = _load_voice(engine, voice_files[53])
    made.voices.append(own)
    sid = made.session(own)
    engine.session_push(sid, chunks[0])
    engine.session_set_voice(sid, vb)
    engine.voice_destroy(made.voices.pop())                          # nothing uses the old voice any more
    _refused(engine, lambda: engine.voice_destroy(vb), 'in use')
    engine.session_push(sid, chunks[1])
    # A -> B -> A cycles, alone and as a member of a mixed group
    alone = made.session(va)
    m, other = made.session(va), made.session(vb)
    gid = made.group([m, other])
    bufs = [np.empty(engine.session_io_geometry(m)['max_out']) for _ in range(2)]
    free = {}
    for cycle in range(1, 13):
        for v in (vb, va):
            engine.session_set_voice(alone, v)
            engine.session_push(alone, chunks[cycle % 3])
            engine.session_set_voice(m, v if v == va else vc)
            engine.group_collect(gid, engine.group_submit(gid, [chunks[cycle % 3]] * 2), bufs)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 switch cycles of a session alone and of a group member')
    assert abs(grown) < 4.0
