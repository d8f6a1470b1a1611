"""Several target voices on one engine (ryk_voice_*, ryk_session_create_voice) and mixed-voice groups whose one batched stage-2
forward reads each member's weights from that member's voice.

  * ungrouped sessions on voices 1 and 2 match the oracle stream of their own model files, and differ from each other;
  * a mixed group's member output is BITWISE the output of the same slot of a homogeneous group on that member's voice (the tile
    grid, K order and split-K depend only on the shapes), through submit / collect and through push_device, and matches its
    voice's oracle; a mixed step launches as many kernels as a homogeneous one;
  * refused groups and voice calls fail with a message and launch nothing; voice create / load / destroy cycles return the memory.

The voices are created on the shared engine from their own seeded model files and destroyed at the end; voice 0 is untouched.
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()
TOL = 1e-3                  # headline tolerance: sample RMSE


def _cfg(T, extra=(0.0, 0.5, 0.0)):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                         buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                         threshold_db=60.0, vocoder_buffer_size=1024)


def _rmse(a, b):
    return float(np.sqrt(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2)))


def _load_voice(engine, paths):
    from realtime_yukarin_b200.models import load_voice
    v = engine.voice_create()
    load_voice(engine, v, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                     'target_statistics_path')})
    return v


@pytest.fixture(scope='module')
def voice_files(tmp_path_factory):
    """Three base-64 voices (seeds 11..13) and two base-16 ones (seeds 14, 15), none shared with the other test modules."""
    out = {}
    for seed in (11, 12, 13):
        out[seed] = synthetic.write_synthetic_models(tmp_path_factory.mktemp(f'voice{seed}'), seed=seed)
    for seed in (14, 15):
        out[seed] = synthetic.write_synthetic_models(tmp_path_factory.mktemp(f'voice{seed}'), seed=seed, base1=16, base2=16)
    return out


@pytest.fixture(scope='module')
def voices(engine, voice_files):
    """voice id -> model paths for the three base-64 voices, loaded on the shared engine; destroyed afterwards."""
    engine.set_precision('fp16')
    ids = {_load_voice(engine, voice_files[seed]): voice_files[seed] for seed in (11, 12, 13)}
    yield ids
    for v in ids:
        engine.voice_destroy(v)


def _oracle_stream(paths, x, T, nchunks, extra=(0.0, 0.5, 0.0)):
    from realtime_yukarin_b200.models import F0Converter
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
    orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
    n = round(T * 24000)
    return [orc.push(x[k * n:(k + 1) * n]) for k in range(nchunks)]


def _run_group_host(engine, voice_of, xs, T, nchunks):
    """A fresh group of one session per entry of voice_of, fed xs[i] through group_submit / collect (3 in flight).
    Returns (per-member list of per-step outputs, launches of the steps)."""
    sids = [engine.session_create(_cfg(T), voice=v) for v in voice_of]
    gid = engine.group_create(sids)
    n = round(T * 24000)
    bufs = [[np.empty(65536) for _ in sids] for _ in range(8)]
    outs = [[] for _ in sids]
    tickets = []

    def collect():
        t = tickets.pop(0)
        for i, o in enumerate(engine.group_collect(gid, t, bufs[t % 8])):
            outs[i].append(o.copy())
    before = engine.launch_count
    for k in range(nchunks):
        tickets.append(engine.group_submit(gid, [x[k * n:(k + 1) * n] for x in xs]))
        if len(tickets) > 3:
            collect()
    while tickets:
        collect()
    launches = engine.launch_count - before
    engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    return outs, launches


def _run_group_device(engine, voice_of, xs, T, nchunks):
    """As _run_group_host through group_push_device (device buffers, one step at a time)."""
    import torch
    sids = [engine.session_create(_cfg(T), voice=v) for v in voice_of]
    gid = engine.group_create(sids)
    n = round(T * 24000)
    cap = engine.session_io_geometry(sids[0])['max_out']
    dev = torch.device('cuda', engine.device)
    outs_d = [torch.zeros(cap, dtype=torch.float64, device=dev) for _ in sids]
    ns_d = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in sids]
    outs = [[] for _ in sids]
    for k in range(nchunks):
        ws = [torch.from_numpy(np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32)).to(dev) for x in xs]
        torch.cuda.synchronize(dev)
        engine.group_push_device(gid, [w.data_ptr() for w in ws], n, [o.data_ptr() for o in outs_d], cap, [c.data_ptr() for c in ns_d])
        engine.synchronize()
        for i in range(len(sids)):
            outs[i].append(outs_d[i][:int(ns_d[i].item())].cpu().numpy().copy())
    engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    return outs


def test_ungrouped_sessions_convert_into_their_voices(engine, voices):
    ids = list(voices)[:2]
    T, nchunks = 0.3, 8
    x = synthetic.synthetic_speech(2.4, stream=81)
    n = round(T * 24000)
    got = {}
    for v in ids:
        sid = engine.session_create(_cfg(T), voice=v)
        assert engine.session_voice(sid) == v
        buf = np.empty(65536)
        tickets, outs = [], []
        for k in range(nchunks):
            tickets.append(engine.session_submit(sid, x[k * n:(k + 1) * n]))
            if len(tickets) > 3:
                outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
        while tickets:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
        engine.session_destroy(sid)
        refs = _oracle_stream(voices[v], x, T, nchunks)
        assert [len(o) for o in outs] == [len(r) for r in refs]
        y, r = np.concatenate(outs), np.concatenate(refs)
        err = _rmse(y, r)
        print(f'voice {v}: {len(y)} samples rmse {err:.3e} signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
        assert err <= TOL
        got[v] = y
    apart = _rmse(got[ids[0]], got[ids[1]])
    print(f'voices {ids[0]} and {ids[1]} differ by rmse {apart:.3e}')
    assert apart > 10 * TOL


@pytest.mark.parametrize('T,pattern,nchunks', [(0.3, (0, 1, 0, 1), 6), (1.0, (0, 1, 2, 0, 1, 2, 2, 0), 3)])
def test_mixed_group_is_bitwise_the_homogeneous_groups(engine, voices, T, pattern, nchunks):
    ids = list(voices)
    voice_of = [ids[p] for p in pattern]
    B = len(voice_of)
    xs = [synthetic.synthetic_speech(nchunks * T + 0.1, stream=90 + i) for i in range(B)]
    mixed, mixed_launches = _run_group_host(engine, voice_of, xs, T, nchunks)
    mixed_dev = _run_group_device(engine, voice_of, xs, T, nchunks)
    for v in sorted(set(voice_of)):
        homo, homo_launches = _run_group_host(engine, [v] * B, xs, T, nchunks)
        homo_dev = _run_group_device(engine, [v] * B, xs, T, nchunks)
        assert homo_launches == mixed_launches, (homo_launches, mixed_launches)
        for i in (i for i in range(B) if voice_of[i] == v):
            for k in range(nchunks):
                assert np.array_equal(mixed[i][k], homo[i][k]), (v, i, k)
                assert np.array_equal(mixed_dev[i][k], homo_dev[i][k]), (v, i, k)
                assert np.array_equal(mixed_dev[i][k], mixed[i][k]), (v, i, k)
    for i in range(B):
        refs = _oracle_stream(voices[voice_of[i]], xs[i], T, nchunks)
        assert [len(o) for o in mixed[i]] == [len(r) for r in refs], i
        err = _rmse(np.concatenate(mixed[i]), np.concatenate(refs))
        print(f'T={T} member {i} (voice {voice_of[i]}): rmse {err:.3e}')
        assert err <= TOL


def _refused(engine, call, needle):
    from realtime_yukarin_b200.engine import RykError
    before = engine.launch_count
    with pytest.raises(RykError, match=needle):
        call()
    assert engine.launch_count == before


def test_refusals(engine, voices, voice_files):
    ids = list(voices)
    cfg = _cfg(0.3)
    made_voices, made_sessions = [], []         # destroyed in the end whatever fails: the engine is shared with later modules

    def voice(seed):
        made_voices.append(_load_voice(engine, voice_files[seed]))
        return made_voices[-1]

    def sessions(*vs):
        out = [engine.session_create(cfg, voice=v) for v in vs]
        made_sessions.extend(out)
        return out
    try:
        narrow = voice(14)
        # stage-2 widths differ
        mixed_width = sessions(ids[0], narrow)
        _refused(engine, lambda: engine.group_create(mixed_width), 'same')
        # two base-16 voices: same widths, but their stage-2 nets run layers on kernels that take one voice
        narrow2 = voice(15)
        both_narrow = sessions(narrow, narrow2)
        _refused(engine, lambda: engine.group_create(both_narrow), 'per batch item')
        # more than 8 distinct voices
        many = sessions(narrow, *[voice(14) for _ in range(8)])
        _refused(engine, lambda: engine.group_create(many), 'at most 8')
        # a mixed group in precision 0
        engine.set_precision('fp32')
        try:
            fp32 = sessions(ids[0], ids[1])
            _refused(engine, lambda: engine.group_create(fp32), 'precision')
        finally:
            engine.set_precision('fp16')
        # a voice in use can neither change nor go
        W, scale, shift = np.zeros((64, 9, 3), np.float32), np.ones(64, np.float32), np.zeros(64, np.float32)
        _refused(engine, lambda: engine.voice_destroy(ids[0]), 'in use')
        _refused(engine, lambda: engine.model_set_layer(1, 0, W, scale, shift, voice=ids[0]), 'in use')
        _refused(engine, lambda: engine.stage1_set_stats(*[np.zeros(9)] * 4, voice=ids[0]), 'in use')
        # sessions on a voice without both models, or on no voice at all
        empty = engine.voice_create()
        made_voices.append(empty)
        engine.model_create(1, 9, 9, 64, voice=empty)
        _refused(engine, lambda: engine.session_create(cfg, voice=empty), 'load')
        engine.voice_destroy(made_voices.pop())
        _refused(engine, lambda: engine.session_create(cfg, voice=empty), 'no such voice')
        _refused(engine, lambda: engine.session_create(cfg, voice=10 ** 6), 'no such voice')
    finally:
        for sid in made_sessions:
            engine.session_destroy(sid)
        for v in made_voices:
            engine.voice_destroy(v)


def test_layer_shapes_of_voices_match_the_library(engine, voice_files):
    """engine._unet_layer_shapes (how the Python side checks the model files of voices >= 1) against ryk_model_layer_shape, which
    reports voice 0's nets as the library built them.  Voice 0 keeps the models it has; an empty one gets the base-16 files."""
    from realtime_yukarin_b200.engine import RykError, _unet_layer_shapes
    try:
        engine.model_layer_shape(1, 0), engine.model_layer_shape(2, 0)
    except RykError:
        from realtime_yukarin_b200.models import load_voice
        load_voice(engine, 0, **{k: voice_files[14][k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                                  'target_statistics_path')})
    for stage in (1, 2):
        got = [engine.model_layer_shape(stage, i) for i in range(16)]
        in_ch, base, out_ch = got[0][1], got[0][2], got[15][2]
        assert got == _unet_layer_shapes(stage, in_ch, out_ch, base), stage


def test_voice_cycles_return_device_memory(engine, voices, voice_files):
    import torch
    ids = list(voices)
    cfg = _cfg(0.3)
    chunk = synthetic.synthetic_speech(0.4, stream=7)[:round(0.3 * 24000)]
    free = {}
    for cycle in range(1, 7):
        engine.synchronize()
        before = torch.cuda.mem_get_info()[0]
        v = _load_voice(engine, voice_files[13])
        engine.synchronize()
        if cycle == 1:
            print(f'one base-64 voice takes {(before - torch.cuda.mem_get_info()[0]) / 2**20:.1f} MiB of device memory')
        sid = engine.session_create(cfg, voice=v)
        engine.session_push(sid, chunk)
        sids = [engine.session_create(cfg, voice=w) for w in (v, ids[0])]
        gid = engine.group_create(sids)
        engine.group_submit(gid, [chunk, chunk])
        engine.synchronize()
        engine.group_destroy(gid)
        for s in [sid] + sids:
            engine.session_destroy(s)
        engine.voice_destroy(v)
        if cycle in (2, 6):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[6]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 4 voice cycles')
    assert abs(grown) < 4.0
