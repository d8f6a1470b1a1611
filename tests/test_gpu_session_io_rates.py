"""Sessions at a sound card's rates: streaming resampling into and out of the session on the GPU (DESIGN.md DECIDE R1).

A session at the models' rate fs = 24 kHz that takes its chunks at R_in must give bitwise the outputs of a native-rate session fed
concat(zeros(D), ryk_resample_poly(x)) in n-sample chunks; a session that returns its samples at R_out must return, after step k,
resample_poly(native synthesizer output)[:M_k]."""
import math
from pathlib import Path

import numpy as np
import pytest
import scipy.signal as ss

from realtime_yukarin_b200 import synthetic, wave_io

pytestmark = pytest.mark.gpu

FS, T, K = 24000, 0.3, 12
N = round(FS * T)


def _load(engine, paths):
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    ac = AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=engine)
    SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=engine)
    return ac


def _cfg(fs=FS, fft_length=1024):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=fs, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=fft_length, order=8, alpha=0.466,
                         buffer_time=T, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0, threshold_db=60.0,
                         vocoder_buffer_size=1024)


def _ratio(r_from, r_to):
    g = math.gcd(r_from, r_to)
    return r_to // g, r_from // g


def _device_input(engine, rate, seconds, stream):
    """float32 test signal at `rate`: synthetic speech resampled from 24 kHz."""
    return wave_io.resample(synthetic.synthetic_speech(seconds, stream=stream), FS, rate, engine)


def _model_rate_input(engine, x, rate):
    """concat(zeros(D), ryk_resample_poly(x)): what a session taking x at `rate` analyses."""
    _, _, D = wave_io.stream_input_geometry(rate, FS, T)
    up, down = _ratio(rate, FS)
    y = engine.resample_poly(x, up, down, wave_io.resample_filter(up, down))
    return np.concatenate([np.zeros(D, np.float32), y]).astype(np.float32)


def _host_output(y, rate, counts):
    """resample_poly of the native synthesizer output, cut at M_k after each step (scipy, float64)."""
    up, down = _ratio(FS, rate)
    z = ss.resample_poly(np.concatenate(y), up, down, window=wave_io.resample_filter(up, down) / up)
    M = [wave_io.stream_output_count(int(c), rate, FS) for c in np.cumsum(counts)]
    return z, M


def _run_host(engine, sid, chunks):
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    return [engine.session_push(sid, c, buf).copy() for c in chunks]


def _run_submit(engine, sid, chunks, depth=4):
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    tickets, outs = [], []
    for c in chunks:
        tickets.append(engine.session_submit(sid, c))
        if len(tickets) > depth:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    while tickets:
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    return outs


def _run_device(engine, sid, chunks):
    import torch
    g = engine.session_io_geometry(sid)
    d_in = torch.from_numpy(np.stack(chunks)).cuda()
    d_out = torch.zeros((len(chunks), g['max_out']), dtype=torch.float64, device='cuda')
    d_n = torch.zeros(len(chunks), dtype=torch.int32, device='cuda')
    for k in range(len(chunks)):
        engine.session_push_device(sid, d_in[k].data_ptr(), len(chunks[k]), d_out[k].data_ptr(), g['max_out'], d_n[k:].data_ptr())
    engine.synchronize()
    n = d_n.cpu().numpy()
    out = d_out.cpu().numpy()
    return [out[k, :n[k]].copy() for k in range(len(chunks))]


def _session(engine, rate_in=FS, rate_out=FS):
    sid = engine.session_create(_cfg())
    engine.session_set_input_rate(sid, rate_in)
    engine.session_set_output_rate(sid, rate_out)
    return sid


@pytest.mark.parametrize('rate', [48000, 44100, 16000])
def test_input_side_bitwise_equals_native_session(engine, small_models, rate):
    _load(engine, small_models)
    x = _device_input(engine, rate, K * T + 0.2, stream=5)
    n_in, _, D = wave_io.stream_input_geometry(rate, FS, T)
    chunks = [x[k * n_in:(k + 1) * n_in] for k in range(K)]
    xm = _model_rate_input(engine, x, rate)
    ref_sid = engine.session_create(_cfg())
    ref = _run_host(engine, ref_sid, [xm[k * N:(k + 1) * N] for k in range(K)])
    engine.session_destroy(ref_sid)
    assert sum(len(r) for r in ref) > 0 and np.abs(np.concatenate(ref)).max() > 0
    for run in (_run_submit, _run_host, _run_device):
        sid = _session(engine, rate_in=rate)
        g = engine.session_io_geometry(sid)
        assert (g['n_in'], g['delay_in'], g['in_rate'], g['out_rate']) == (n_in, D, rate, FS)
        got = run(engine, sid, chunks)
        engine.session_destroy(sid)
        assert [len(o) for o in got] == [len(r) for r in ref], run.__name__
        for k, (o, r) in enumerate(zip(got, ref)):
            assert np.array_equal(o, r), (run.__name__, k)


@pytest.mark.parametrize('rate', [48000, 44100])
def test_output_side_matches_resample_poly(engine, small_models, rate):
    _load(engine, small_models)
    x = synthetic.synthetic_speech(K * T + 0.2, stream=6)
    chunks = [x[k * N:(k + 1) * N] for k in range(K)]
    ref_sid = engine.session_create(_cfg())
    y = _run_host(engine, ref_sid, chunks)
    engine.session_destroy(ref_sid)
    z, M = _host_output(y, rate, [len(v) for v in y])
    peak = np.abs(np.concatenate(y)).max()
    assert peak > 0
    for run in (_run_submit, _run_device):
        sid = _session(engine, rate_out=rate)
        max_out = engine.session_io_geometry(sid)['max_out']
        got = run(engine, sid, chunks)
        engine.session_destroy(sid)
        assert [len(o) for o in got] == list(np.diff([0] + M)), run.__name__
        assert max(len(o) for o in got) <= max_out
        cat = np.concatenate(got)
        assert np.abs(cat - z[:M[-1]]).max() <= 1e-12 * peak, run.__name__


def test_group_at_device_rates_equals_native_group(engine, small_models):
    _load(engine, small_models)
    B, rate = 4, 48000
    n_in, _, _ = wave_io.stream_input_geometry(rate, FS, T)
    xs = [_device_input(engine, rate, K * T + 0.2, stream=20 + i) for i in range(B)]
    xms = [_model_rate_input(engine, x, rate) for x in xs]

    def run_group(sids, chunk_of, n):
        gid = engine.group_create(sids)
        cap = max(engine.session_io_geometry(s)['max_out'] for s in sids)
        outs = [np.empty(cap) for _ in sids]
        got = [[] for _ in sids]
        for k in range(K):
            t = engine.group_submit(gid, [chunk_of(i, k) for i in range(B)])
            for i, o in enumerate(engine.group_collect(gid, t, outs)):
                got[i].append(o.copy())
        engine.group_destroy(gid)
        for s in sids:
            engine.session_destroy(s)
        return got

    native = run_group([engine.session_create(_cfg()) for _ in range(B)], lambda i, k: xms[i][k * N:(k + 1) * N], N)
    dev = run_group([_session(engine, rate, rate) for _ in range(B)], lambda i, k: xs[i][k * n_in:(k + 1) * n_in], n_in)
    for i in range(B):
        z, M = _host_output(native[i], rate, [len(v) for v in native[i]])
        assert [len(o) for o in dev[i]] == list(np.diff([0] + M)), i
        peak = np.abs(np.concatenate(native[i])).max()
        assert np.abs(np.concatenate(dev[i]) - z[:M[-1]]).max() <= 1e-12 * peak, i
    # the input side alone is bitwise: a 48 kHz-in / 24 kHz-out group against the native group
    inonly = run_group([_session(engine, rate, FS) for _ in range(B)], lambda i, k: xs[i][k * n_in:(k + 1) * n_in], n_in)
    for i in range(B):
        for k in range(K):
            assert np.array_equal(inonly[i][k], native[i][k]), (i, k)
    # members with different device rates cannot share one chunk length
    a, b = _session(engine, rate, rate), _session(engine, FS, FS)
    c = _session(engine, rate, FS)
    with pytest.raises(Exception, match='same device input and output rates'):
        engine.group_create([a, b])
    with pytest.raises(Exception, match='same device input and output rates'):
        engine.group_create([a, c])
    for s in (a, b, c):
        engine.session_destroy(s)


def test_realtime_pipeline_at_48k(engine, small_models, tmp_path):
    """RealtimePipeline at 48/48 kHz with the device re-blocker plays what the 24 kHz session's synthesizer output, resampled as
    above and re-blocked at 48 kHz by OutputReblocker, gives; run.run(--wav_in) writes a 48 kHz wav of K out_audio_chunks."""
    import yaml
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import Item, OutputReblocker, RealtimePipeline
    ac = _load(engine, small_models)
    rate = 48000
    fields = dict(input_device_name=None, output_device_name=None, input_rate=rate, output_rate=rate, frame_period=5.0, buffer_time=T,
                  vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0, output_silent_threshold=80.0,
                  encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    paths = {k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path', 'stage1_config_path',
                                          'stage2_model_path', 'stage2_config_path')}
    cfg = Config(extract_f0_mode=VocodeMode.WORLD, **fields, **paths)
    x = _device_input(engine, rate, K * T + 0.2, stream=9)
    x[int(1.2 * rate):int(2.4 * rate)] *= 1e-6
    n_in = cfg.in_audio_chunk
    pipe = RealtimePipeline(cfg, acoustic_param=ac.config.dataset.acoustic_param, engine=engine, depth=3)
    for k in range(K):
        pipe.put(Item(item=x[k * n_in:(k + 1) * n_in], index=k))
    pipe.flush()
    got = []
    while True:
        it = pipe.get_nowait()
        if it is None:
            break
        got.append(it)
    pipe.close()
    assert [it.index for it in got] == list(range(K))
    # the same chunks by hand: native session on the model-rate input, host resampling, OutputReblocker at 48 kHz
    xm = _model_rate_input(engine, x, rate)
    sid = engine.session_create(_cfg())
    y = _run_host(engine, sid, [xm[k * N:(k + 1) * N] for k in range(K)])
    engine.session_destroy(sid)
    z, M = _host_output(y, rate, [len(v) for v in y])
    rb = OutputReblocker(cfg.out_audio_chunk, cfg.output_silent_threshold, max_in=max(np.diff([0] + M)) + 1, engine=engine)
    played = 0
    for k, it in enumerate(got):
        ref = rb.push(z[(M[k - 1] if k else 0):M[k]])
        assert (it.item is None) == (ref is None), k
        if ref is not None:
            played += 1
            assert np.abs(it.item - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), k
    rb.close()
    assert played > 0
    # run.py with a 48 kHz config and a 24 kHz wav: the file is resampled on load, the session at 48 kHz writes 48 kHz
    cfg_yaml = dict(fields, extract_f0_mode='world', **{k: str(v) for k, v in paths.items()})
    (tmp_path / 'config.yaml').write_text(yaml.safe_dump(cfg_yaml))
    wav_in = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
    n = run_mod.run(tmp_path / 'config.yaml', wav_in=wav_in, wav_out=tmp_path / 'out.wav', engine=engine, depth=2)
    out, sr = wave_io.read_wav(tmp_path / 'out.wav')
    # one out_audio_chunk per loop iteration, then the chunks still in flight when the file ended
    assert sr == rate and n == len(wave_io.load_wave(wav_in, rate, engine).wave) // n_in
    assert len(out) % cfg.out_audio_chunk == 0 and n * cfg.out_audio_chunk <= len(out) <= (n + 3) * cfg.out_audio_chunk


def test_errors_launch_nothing(engine, small_models):
    """Refused calls fail with a clear message before any kernel is queued."""
    _load(engine, small_models)
    x = synthetic.synthetic_speech(1.0, stream=1)
    sid = engine.session_create(_cfg())
    engine.session_push(sid, x[:N])
    engine.synchronize()

    def refused(call, match):
        before = engine.launch_count
        with pytest.raises(Exception, match=match):
            call()
        assert engine.launch_count == before

    refused(lambda: engine.session_set_input_rate(sid, 48000), 'fresh session')
    refused(lambda: engine.session_set_output_rate(sid, 48000), 'fresh session')
    engine.session_destroy(sid)
    c = _cfg()
    c.buffer_time = 0.005                       # 120 samples at 24 kHz; round(220.5) = 220 at 44.1 kHz is not whole
    sid = engine.session_create(c)
    refused(lambda: engine.session_set_input_rate(sid, 44100), 'not a whole number')
    engine.session_destroy(sid)
    # the synthesizer at 48 kHz would read 1025-bin rows out of a 513-bin decode window
    refused(lambda: engine.session_create(_cfg(fs=48000, fft_length=1024)), 'fs does not match fft_length')


def test_device_rate_sessions_free_their_memory(engine, small_models):
    import torch
    _load(engine, small_models)
    x = _device_input(engine, 48000, 1.0, stream=5)
    n_in = round(48000 * T)
    free = {}
    for cycle in range(1, 21):
        sid = _session(engine, 48000, 44100)
        engine.session_push(sid, x[:n_in])
        engine.session_destroy(sid)
        if cycle in (5, 20):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    assert abs(free[5] - free[20]) / 2**20 < 4.0
