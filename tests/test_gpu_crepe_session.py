"""CREPE f0 mode inside the device-resident session (ryk_engine_set_f0_method(e, 2), csrc/crepe.cu CrepePlan): each step's encode
window is resampled to 16 kHz, run through the network and decoders and the voicing rule on the device, and its f0 replaces
DIO/StoneMask in the captured analysis graph.  In precision 1 the CREPE convolutions run on the 3xTF32 tensor-core kernel
(csrc/crepe_tc.cu), checked here layer by layer and through the whole network.  Checked against the host-class chain with Vocoder(extract_f0_mode=CREPE), which
analyses the same windows through ryk_crepe_predict, and through the public RealtimePipeline with extract_f0_mode: crepe."""
import dataclasses

import numpy as np
import pytest

from realtime_yukarin_b200 import crepe as pcrepe
from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import RykError, SessionConfig

from .test_gpu_parity import _load, _speech

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def crepe_tiny(tmp_path_factory):
    return synthetic.write_crepe_model(tmp_path_factory.mktemp('crepe_tiny'), seed=5, capacity='tiny')


@pytest.fixture(scope='module')
def crepe_full(tmp_path_factory):
    return synthetic.write_crepe_model(tmp_path_factory.mktemp('crepe_full'), seed=6, capacity='full')


def _layer_shapes(capacity):
    """(Win, Cin, Cout, k) of CREPE conv layers 1..6 as the network runs them: layer 1 as the 1x1 GEMM over its im2col rows, layers
    2..6 over the zero-framed ('same' padding) inputs."""
    m = pcrepe.CAPACITY[capacity]
    cout = [f * m for f in (32, 4, 4, 4, 8, 16)]
    shapes, w = [(256, 512, cout[0], 1)], 128
    for l in range(1, 6):
        shapes.append((w + 63, cout[l - 1], cout[l], 64))
        w //= 2
    return shapes


@pytest.mark.parametrize('capacity', ['tiny', 'full'])
@pytest.mark.parametrize('F', [1, 61, 201])
def test_crepe_tc_conv_layers(engine, capacity, F):
    """3xTF32 tensor-core kernel on every conv layer shape against a float64 torch reference on the device.  Error of each output is
    normalised by sum |a * w| over its inputs.  Bound: at most 8x the FP32 CUDA-core kernel's worst normalised error on the same layer.
    Each 3xTF32 product keeps hi*hi + hi*lo + lo*hi of operands rounded to 11 + 11 significant bits, so a product is exact to about
    2^-21 relative instead of FP32's 2^-24 (a factor 8); the FP32 accumulation is common to both kernels.  Also bitwise determinism."""
    import torch
    rng = np.random.default_rng(100 * F + len(capacity))
    for i, (Win, Cin, Cout, k) in enumerate(_layer_shapes(capacity)):
        x = rng.standard_normal((F, Win, Cin)).astype(np.float32)
        W = (rng.standard_normal((Cout, Cin, k)) / np.sqrt(Cin * k)).astype(np.float32)
        b = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
        xt = torch.from_numpy(x).cuda().double().permute(0, 2, 1)
        Wt = torch.from_numpy(W).cuda().double()
        ref = torch.relu(torch.nn.functional.conv1d(xt, Wt, torch.from_numpy(b).cuda().double())).permute(0, 2, 1)
        mag = torch.nn.functional.conv1d(xt.abs(), Wt.abs()).permute(0, 2, 1) + abs(torch.from_numpy(b).cuda().double())
        errs = {}
        for backend in (0, 1):
            y = torch.from_numpy(pcrepe.run_test_conv(engine, backend, x, W, b)).cuda().double()
            errs[backend] = float(((y - ref).abs() / mag).max())
        y1 = pcrepe.run_test_conv(engine, 1, x, W, b)
        y2 = pcrepe.run_test_conv(engine, 1, x, W, b)
        assert np.array_equal(y1, y2), (capacity, F, i)
        print(f'crepe {capacity} layer {i + 1} F={F} ({Win}x{Cin} -> {Cout}, k {k}): normalised max err fp32 {errs[0]:.2e}, 3xtf32 {errs[1]:.2e}')
        assert errs[1] <= 8 * errs[0] + 1e-9, (capacity, F, i, errs)


@pytest.mark.parametrize('capacity,seconds', [('tiny', 0.9), ('full', 0.3)])
def test_crepe_tc_network_and_decoders_match_oracle(engine, tmp_path, capacity, seconds):
    """Mode-1 (3xTF32) activations against the oracle within the 5e-4 of the FP32 CREPE test; the device decoders applied to them
    give exactly the oracle decoders' path and voicing."""
    from oracle import crepe as oc
    from scipy.signal import resample_poly
    w = synthetic.make_crepe_params(3, capacity)
    path = tmp_path / 'crepe.npz'
    np.savez(path, **w)
    pcrepe.load_crepe_model(path, engine)
    x16 = resample_poly(_speech(seconds, 21).astype(np.float64), 2, 3).astype(np.float32)
    act, ppath, voicing, _ = pcrepe.run_test_network(engine, 1, x16, 5.0)
    act_ref = oc.get_activation(x16, w, 5.0)
    err = float(np.abs(act - act_ref).max())
    print(f'crepe {capacity} 3xtf32: {act.shape[0]} frames, activation max |err| {err:.2e}')
    assert err < 5e-4
    _, path_ref = oc.to_viterbi_cents(act)
    assert np.array_equal(ppath, path_ref)
    assert np.array_equal(voicing, oc.predict_voicing(act.max(1)))


def _cfg(T, extra):
    return SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                         buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                         threshold_db=60.0, vocoder_buffer_size=1024)


def _crepe_session(engine, cfg):
    prev = engine.f0_method
    engine.set_f0_method('crepe')
    try:
        return engine.session_create(cfg)
    finally:
        engine.set_f0_method(prev)


def _push_all(engine, sid, x, n):
    return [engine.session_push(sid, x[k * n:(k + 1) * n]).copy() for k in range(len(x) // n)]


def _rmse(a, b):
    return float(np.sqrt(np.mean((np.concatenate(a) - np.concatenate(b)) ** 2)))


@pytest.mark.parametrize('T,extra', [(0.3, (0.0, 0.5, 0.0)), (0.1, (0.1, 0.2, 0.0)), (1.0, (0.0, 0.5, 0.0))])
def test_crepe_session_matches_host_chain(engine, small_models, crepe_tiny, T, extra):
    """fp32 CREPE session == EncodeStream / ConvertStream / DecodeStream with Vocoder(extract_f0_mode=CREPE), sample RMSE < 1e-3."""
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.params import create_from_json
    from realtime_yukarin_b200.stream import ConvertStream, DecodeStream, EncodeStream, StreamWrapper
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    ac, sr, _ = _load(engine, small_models)
    pcrepe.load_crepe_model(crepe_tiny, engine)
    acp = create_from_json(small_models['stage1_config_path']).dataset.acoustic_param
    engine.set_precision('fp32')
    voc = RealtimeVocoder(acoustic_param=acp, out_sampling_rate=24000, extract_f0_mode=VocodeMode.CREPE)
    voc.create_synthesizer(buffer_size=1024, number_of_pointers=16)
    es, cs, ds = EncodeStream(voc), ConvertStream(VoiceChanger(ac, sr, threshold=60)), DecodeStream(voc)
    ws = [StreamWrapper(es, extra[0]), StreamWrapper(cs, extra[1]), StreamWrapper(ds, extra[2])]
    x = _speech(2.4 if T < 1.0 else 4.0, 52)
    n = round(T * 24000)
    refs = []
    for k in range(len(x) // n):
        es.add(start_time=extra[0] + k * T, data=x[k * n:(k + 1) * n])
        cs.add(start_time=extra[1] + k * T, data=ws[0].process_next(T))
        ds.add(start_time=extra[2] + k * T, data=ws[1].process_next(T))
        refs.append(ws[2].process_next(T))
    sid = _crepe_session(engine, _cfg(T, extra))
    outs = _push_all(engine, sid, x, n)
    engine.session_destroy(sid)
    engine.set_precision('fp16')
    assert [len(o) for o in outs] == [len(r) for r in refs]
    rmse = _rmse(outs, refs)
    print(f'crepe session T={T} extra={extra}: {sum(map(len, outs))} samples, rmse {rmse:.3e}')
    assert rmse < 1e-3


@pytest.mark.parametrize('precision', ['fp32', 'fp16'])
def test_crepe_session_pipelined_equals_sequential(engine, small_models, crepe_tiny, precision):
    _load(engine, small_models)
    pcrepe.load_crepe_model(crepe_tiny, engine)
    engine.set_precision(precision)
    T, n = 0.3, 7200
    x = _speech(3.6, 44)
    sid = _crepe_session(engine, _cfg(T, (0.0, 0.5, 0.0)))
    seq = _push_all(engine, sid, x, n)
    engine.session_destroy(sid)
    sid = _crepe_session(engine, _cfg(T, (0.0, 0.5, 0.0)))
    buf, tickets, outs = np.empty(32768), [], []
    for k in range(len(x) // n):
        tickets.append(engine.session_submit(sid, x[k * n:(k + 1) * n]))
        if len(tickets) > 4:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    while tickets:
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    engine.session_destroy(sid)
    engine.set_precision('fp16')
    assert len(outs) == len(seq)
    for a, b in zip(outs, seq):
        assert np.array_equal(a, b)


def test_crepe_session_full_capacity_precision1(engine, small_models, crepe_full):
    """Precision 1 runs the CREPE convolutions on the 3xTF32 kernel: finite output, identical across two sessions."""
    _load(engine, small_models)
    pcrepe.load_crepe_model(crepe_full, engine)
    x, n = _speech(2.4, 61), 7200
    res = {}
    for precision in ('fp16', 'fp16', 'fp32'):
        engine.set_precision(precision)
        sid = _crepe_session(engine, _cfg(0.3, (0.0, 0.5, 0.0)))
        res.setdefault(precision, []).append(np.concatenate(_push_all(engine, sid, x, n)))
        engine.session_destroy(sid)
    engine.set_precision('fp16')
    a, b = res['fp16']
    assert np.all(np.isfinite(a)) and np.array_equal(a, b)
    print(f'crepe full fp16 session vs fp32 session: rmse {float(np.sqrt(np.mean((a - res["fp32"][0]) ** 2))):.3e}')


def test_realtime_pipeline_crepe_mode(engine, small_models, crepe_tiny, monkeypatch):
    """extract_f0_mode: crepe selects the CREPE session (weights from RYK_CREPE_MODEL); the engine's f0 method is restored."""
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.worker import OutputReblocker, RealtimePipeline
    from .test_gpu_widen import _config
    ac, _, _ = _load(engine, small_models)
    acp = ac.config.dataset.acoustic_param
    engine.set_precision('fp32')
    cfg = dataclasses.replace(_config(small_models, 0.3, 80.0), extract_f0_mode=VocodeMode.CREPE)
    monkeypatch.setitem(pcrepe._loaded, 'engine', None)
    monkeypatch.delenv('RYK_CREPE_MODEL', raising=False)
    with pytest.raises(RuntimeError, match='no CREPE weights loaded'):
        RealtimePipeline(cfg, acoustic_param=acp, engine=engine)
    assert engine.f0_method == 'dio'
    monkeypatch.setenv('RYK_CREPE_MODEL', str(crepe_tiny))
    pipe = RealtimePipeline(cfg, acoustic_param=acp, engine=engine, depth=2)
    assert engine.f0_method == 'dio'
    x, n = _speech(3.0, 8), cfg.in_audio_chunk
    got = [pipe.process(x[k * n:(k + 1) * n], block=True) for k in range(len(x) // n)]
    pipe.close()
    sid = _crepe_session(engine, _cfg(0.3, (0.0, 0.5, 0.0)))
    rb = OutputReblocker(cfg.out_audio_chunk, cfg.output_silent_threshold, engine=engine)
    want = []
    for k in range(len(x) // n):
        c = rb.push(engine.session_push(sid, x[k * n:(k + 1) * n] * cfg.input_scale))
        want.append(np.zeros(n, np.float32) if c is None else (c * cfg.output_scale).astype(np.float32))
    rb.close()
    engine.session_destroy(sid)
    engine.set_precision('fp16')
    assert any(w.any() for w in want)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_crepe_session_errors_memory_and_group(engine, small_models, crepe_tiny):
    import torch
    _load(engine, small_models)
    pcrepe.load_crepe_model(crepe_tiny, engine)
    cfg = _cfg(0.3, (0.0, 0.5, 0.0))
    x, n = _speech(2.4, 17), 7200
    # the model may not change under a live CREPE session; it may again once the session is gone
    sid = _crepe_session(engine, cfg)
    with pytest.raises(RykError, match='in use by a live session'):
        pcrepe.load_crepe_model(crepe_tiny, engine)
    engine.session_destroy(sid)
    pcrepe.load_crepe_model(crepe_tiny, engine)
    # single-signal WORLD f0 is not available in method 2
    engine.set_f0_method('crepe')
    try:
        with pytest.raises(RykError, match='sessions only'):
            engine.world_f0(x[:n], 24000, 5.0, 71.0, 800.0)
    finally:
        engine.set_f0_method('dio')
    # create / push / destroy does not grow device memory
    free = {}
    for cycle in range(1, 21):
        sid = _crepe_session(engine, cfg)
        engine.session_push(sid, x[:n])
        engine.session_destroy(sid)
        if cycle in (5, 20):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[5] - free[20]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 15 CREPE session cycles')
    assert abs(grown) < 4.0
    # a group of two CREPE sessions == the ungrouped sessions (fp32)
    engine.set_precision('fp32')
    xs = [_speech(2.4, 80 + i) for i in range(2)]
    single = []
    for xi in xs:
        sid = _crepe_session(engine, cfg)
        single.append(_push_all(engine, sid, xi, n))
        engine.session_destroy(sid)
    sids = [_crepe_session(engine, cfg) for _ in range(2)]
    gid = engine.group_create(sids)
    bufs = [np.empty(32768) for _ in range(2)]
    grouped = [[], []]
    for k in range(len(xs[0]) // n):
        t = engine.group_submit(gid, [xi[k * n:(k + 1) * n] for xi in xs])
        for i, o in enumerate(engine.group_collect(gid, t, bufs)):
            grouped[i].append(o.copy())
    engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    engine.set_precision('fp16')
    for i in range(2):
        assert [len(o) for o in grouped[i]] == [len(o) for o in single[i]]
        rmse = _rmse(grouped[i], single[i])
        print(f'crepe group member {i}: rmse vs ungrouped {rmse:.3e}')
        assert rmse < 1e-3
