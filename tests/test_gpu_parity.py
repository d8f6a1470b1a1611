"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances (stated per north_star: "per-frame spectral L2 and sample RMSE"):
  * f0 / voiced / silence mask / pulse positions: exact decisions, f0 values within 1e-9 relative (FP64 both sides)
  * sp, ap, mc (FP64 math, FP32 storage): 1e-5 relative
  * stage 1 (FP32 CUDA cores): 2e-4 absolute on O(1) features
  * stage 2 FP32 mode: 1e-3 in the log-spectrum; FP16 tensor-core mode: 3e-2 in the log-spectrum (per-frame L2 / sqrt(bins))
  * waveform: sample RMSE <= 1e-3 (FP32 mode), reported for the FP16 mode
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import synthetic

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()


def _speech(seconds=0.6, stream=0):
    return synthetic.synthetic_speech(seconds, stream=stream)


def test_world_analysis_matches_oracle(engine):
    for stream, seconds in ((0, 0.3), (1, 1.0), (2, 0.1)):
        x = _speech(seconds, stream)
        ref = opipe.extract_features(x, CFG)
        got = engine.world_analyze(x, CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil, CFG.fft_length, CFG.order, CFG.alpha)
        f0r, f0g = ref['f0'].ravel(), got['f0']
        assert np.array_equal(f0r != 0, f0g != 0), (f0r, f0g)
        assert np.allclose(f0g, f0r, rtol=1e-6, atol=0)
        assert np.array_equal(ref['voiced'].ravel(), got['voiced'])
        assert np.allclose(np.log(got['sp']), np.log(ref['sp']), atol=2e-4), np.abs(np.log(got['sp']) - np.log(ref['sp'])).max()
        assert np.allclose(got['ap'], ref['ap'], rtol=1e-4, atol=1e-6), np.abs(got['ap'] - ref['ap']).max()
        assert np.allclose(got['mc'], ref['mc'], atol=2e-4), np.abs(got['mc'] - ref['mc']).max()


def test_world_f0_double_precision(engine):
    x = _speech(1.0, 5)
    f0_ref, t = oworld.dio(x.astype(np.float64), CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil)
    f0_ref = oworld.stonemask(x.astype(np.float64), CFG.fs, t, f0_ref)
    f0, tt = engine.world_f0(x, CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil)
    assert np.array_equal(f0 != 0, f0_ref != 0)
    assert np.allclose(f0, f0_ref, rtol=1e-9)
    assert np.allclose(tt, t)


def test_silence_mask_and_mc2sp(engine):
    x = _speech(1.3, 3)
    n_frames = len(x) // CFG.hop
    for thr in (60.0, 30.0, None):
        ref = opipe.effective_mask(x, n_frames, CFG, thr)
        got = engine.silence_mask(x, CFG.fft_length, CFG.hop, thr, n_frames)
        assert np.array_equal(ref, got)
    rng = np.random.default_rng(0)
    mc = (synthetic.MC_MEAN_OUT + synthetic.MC_STD_OUT * rng.standard_normal((50, 9))).astype(np.float32)
    ref = oworld.mc2sp(mc, CFG.alpha, CFG.fft_length)
    got = engine.mc2sp(mc, CFG.alpha, CFG.fft_length)
    assert np.allclose(np.log(got), np.log(ref), atol=1e-9)


def _load(engine, paths):
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    ac = AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=engine)
    sr = SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=engine)
    return ac, sr, f0c


def test_stage1_matches_oracle(engine, small_models, full_models):
    rng = np.random.default_rng(1)
    for paths in (small_models, full_models):
        ac, sr, f0c = _load(engine, paths)
        p1 = onets.load_npz(paths['stage1_model_path'])
        for T in (60, 128, 260):
            mc = (synthetic.MC_MEAN_IN + synthetic.MC_STD_IN * rng.standard_normal((T, 9))).astype(np.float32)
            ref = onets.stage1_convert(mc, p1, backend='torch')
            engine.set_precision('fp32')
            got = engine.stage1_convert(mc)
            engine.set_precision('fp16')
            got16 = engine.stage1_convert(mc)
            err, err16 = np.abs(got - ref).max(), np.abs(got16 - ref).max()
            print(f'stage1 T={T}: fp32 max err {err:.2e}; fp16-tc max err {err16:.2e} (feature std ~0.1-0.9)')
            assert err < 5e-4, (T, err)
            assert err16 < 2e-2, (T, err16)


def _logspec_err(a, b):
    d = np.log(a.astype(np.float64)) - np.log(b.astype(np.float64))
    return float(np.sqrt((d ** 2).mean(axis=1)).max()), float(np.abs(d).max())


def test_stage2_fp32_and_fp16_match_oracle(engine, small_models, full_models):
    rng = np.random.default_rng(2)
    for paths, Ts in ((small_models, (60, 260)), (full_models, (100,))):
        ac, sr, f0c = _load(engine, paths)
        p2 = onets.load_npz(paths['stage2_model_path'])
        for T in Ts:
            sp = np.exp(-9 + 2.5 * rng.standard_normal((T, 513))).astype(np.float32)
            ref = onets.stage2_convert(sp, p2, backend='torch')
            engine.set_precision('fp32')
            got32 = engine.stage2_convert(sp)
            engine.set_precision('fp16')
            got16 = engine.stage2_convert(sp)
            l2_32, mx_32 = _logspec_err(got32, ref)
            l2_16, mx_16 = _logspec_err(got16, ref)
            print(f'stage2 T={T}: fp32 per-frame L2 {l2_32:.2e} max {mx_32:.2e}; fp16-tc L2 {l2_16:.2e} max {mx_16:.2e}')
            assert l2_32 < 1e-3 and mx_32 < 5e-3
            assert l2_16 < 3e-2 and mx_16 < 0.25


def test_synthesizer_matches_oracle(engine):
    x = _speech(1.2, 7)
    f = opipe.extract_features(x, CFG)
    fft = oworld.cheaptrick_fft_size(CFG.fs)
    ref_s = oworld.RealtimeSynthesizer(CFG.fs, CFG.frame_period, fft, 1024)
    sid = engine.synth_create(CFG.fs, CFG.frame_period, fft, 1024)
    total_ref, total_got = [], []
    for a in range(0, len(f['f0']), 60):
        sl = slice(a, a + 60)
        f0 = f['f0'][sl].ravel().astype(np.float64)
        yr = ref_s.decode(f0, f['sp'][sl], f['ap'][sl])
        yg = engine.synth_decode(sid, f0, f['sp'][sl], f['ap'][sl])
        assert len(yr) == len(yg), (len(yr), len(yg))
        total_ref.append(yr)
        total_got.append(yg)
    yr, yg = np.concatenate(total_ref), np.concatenate(total_got)
    assert len(yr) > 0
    rmse = float(np.sqrt(np.mean((yr - yg) ** 2)))
    print('synth rmse', rmse, 'rms', float(np.sqrt(np.mean(yr ** 2))))
    assert rmse < 1e-6 * max(1.0, float(np.abs(yr).max()) * 1e3)


def test_synthesizer_add_and_synthesis2_equal_decode(engine):
    # the world4py call pattern (AddParameters, then Synthesis2 until it has no block) is bitwise one decode of the same frames
    x = _speech(1.2, 7)
    f = opipe.extract_features(x, CFG)
    fft = oworld.cheaptrick_fft_size(CFG.fs)
    sid_dec = engine.synth_create(CFG.fs, CFG.frame_period, fft, 1024)
    sid_blk = engine.synth_create(CFG.fs, CFG.frame_period, fft, 1024)
    n_blocks = 0
    for a in range(0, len(f['f0']), 60):
        sl = slice(a, a + 60)
        f0 = f['f0'][sl].ravel().astype(np.float64)
        yd = engine.synth_decode(sid_dec, f0, f['sp'][sl], f['ap'][sl])
        assert engine.synth_add_parameters(sid_blk, f0, f['sp'][sl], f['ap'][sl]) == 1
        blocks = []
        while (b := engine.synth_synthesis2(sid_blk)) is not None:
            blocks.append(b)
        yb = np.concatenate(blocks) if blocks else np.zeros(0)
        assert np.array_equal(yd, yb), (a, len(yd), len(yb))
        n_blocks += len(blocks)
    assert n_blocks > 0
    engine.synth_destroy(sid_dec)
    engine.synth_destroy(sid_blk)


def test_synthesizer_nan_on_silent_frames(engine):
    fft = oworld.cheaptrick_fft_size(CFG.fs)
    nb = fft // 2 + 1
    ref_s = oworld.RealtimeSynthesizer(CFG.fs, CFG.frame_period, fft, 1024)
    sid = engine.synth_create(CFG.fs, CFG.frame_period, fft, 1024)
    f0 = np.zeros(60)
    sp = np.zeros((60, nb), np.float32)
    ap = np.zeros((60, nb), np.float32)
    for _ in range(2):
        yr = ref_s.decode(f0, sp, ap)
        yg = engine.synth_decode(sid, f0, sp, ap)
        assert len(yr) == len(yg)
        assert np.array_equal(np.isnan(yr), np.isnan(yg))


def test_convert_window_fused_and_staged(engine, small_models):
    from realtime_yukarin_b200.feature import AcousticFeatureWrapper, Wave
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    x = _speech(1.3, 11)
    enc = opipe.extract_features(x, CFG)
    ref = opipe.convert_window(x, enc, CFG, p1, p2, f0c.stats(), backend='torch')
    engine.set_precision('fp32')
    fw = AcousticFeatureWrapper(wave=Wave(x, CFG.fs), f0=enc['f0'], ap=enc['ap'], mc=enc['mc'], voiced=enc['voiced'])
    for fused in (False, True):
        vc = VoiceChanger(ac, sr, threshold=60, fused=fused)
        out = vc.convert_from_acoustic_feature(fw)
        assert np.array_equal(out.voiced.ravel(), ref['voiced'].ravel())
        assert np.allclose(out.f0.ravel(), ref['f0'].ravel(), rtol=1e-6)
        assert np.allclose(out.ap, ref['ap'])
        l2, mx = _logspec_err(out.sp, ref['sp'])
        print('convert_window fused' if fused else 'convert_window staged', l2, mx)
        assert l2 < 2e-3
    engine.set_precision('fp16')


def test_stream_api_end_to_end(engine, small_models):
    """check.py-style chunked run through EncodeStream/ConvertStream/DecodeStream vs the oracle stream."""
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.params import create_from_json
    from realtime_yukarin_b200.stream import ConvertStream, DecodeStream, EncodeStream, StreamWrapper
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    acp = create_from_json(small_models['stage1_config_path']).dataset.acoustic_param
    T, extra = 0.3, (0.0, 0.5, 0.0)
    for precision, tol in (('fp32', 1e-3), ('fp16', None)):
        engine.set_precision(precision)
        voc = RealtimeVocoder(acoustic_param=acp, out_sampling_rate=24000, extract_f0_mode=VocodeMode.WORLD)
        voc.create_synthesizer(buffer_size=1024, number_of_pointers=16)
        es, cs, ds = EncodeStream(voc), ConvertStream(VoiceChanger(ac, sr, threshold=60)), DecodeStream(voc)
        ws = [StreamWrapper(es, extra[0]), StreamWrapper(cs, extra[1]), StreamWrapper(ds, extra[2])]
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        x = _speech(2.4, 21)
        n = round(T * 24000)
        outs, refs = [], []
        for k in range(len(x) // n):
            chunk = x[k * n:(k + 1) * n]
            es.add(start_time=extra[0] + k * T, data=chunk)
            f = ws[0].process_next(T)
            cs.add(start_time=extra[1] + k * T, data=f)
            c = ws[1].process_next(T)
            ds.add(start_time=extra[2] + k * T, data=c)
            outs.append(ws[2].process_next(T))
            refs.append(orc.push(chunk))
            assert len(outs[-1]) == len(refs[-1])
        y, r = np.concatenate(outs), np.concatenate(refs)
        rmse = float(np.sqrt(np.mean((y - r) ** 2)))
        rms = float(np.sqrt(np.mean(r ** 2)))
        print(f'end-to-end {precision}: samples {len(y)} rmse {rmse:.3e} signal rms {rms:.3e}')
        if tol is not None:
            assert rmse < tol
    engine.set_precision('fp16')


def test_device_session_matches_oracle_stream(engine, small_models):
    """The device-resident session (sliding windows in HBM) == the oracle's chunked stream."""
    from realtime_yukarin_b200.engine import SessionConfig
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    # BASELINE.json configs: [1] 0.3 s / (0,0.5,0); [2] buffer sweep 0.1 / 0.3 / 1.0 s with overlaps; [0] check.py's 1 s chunks with (0,1,0)
    for T, extra in ((0.3, (0.0, 0.5, 0.0)), (0.1, (0.1, 0.2, 0.0)), (0.1, (0.0, 0.5, 0.0)), (1.0, (0.0, 0.5, 0.0)), (1.0, (0.0, 1.0, 0.0)),
                     (0.3, (0.1, 0.5, 0.1))):
        engine.set_precision('fp32')
        cfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                            buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                            threshold_db=60.0, vocoder_buffer_size=1024)
        sid = engine.session_create(cfg)
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        x = _speech(2.4 if T < 1.0 else 5.0, 33)
        n = round(T * 24000)
        outs, refs = [], []
        for k in range(len(x) // n):
            y = engine.session_push(sid, x[k * n:(k + 1) * n])
            r = orc.push(x[k * n:(k + 1) * n])
            assert len(y) == len(r), (k, len(y), len(r))
            outs.append(y.copy())
            refs.append(r)
        y, r = np.concatenate(outs), np.concatenate(refs)
        rmse = float(np.sqrt(np.mean((y - r) ** 2)))
        print(f'session T={T} extra={extra}: {len(y)} samples, rmse {rmse:.3e}, signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
        if rmse >= 1e-3:      # diagnostics: which chunks differ, and by how much
            per = [(k, len(a), float(np.sqrt(np.mean((a - b) ** 2))) if len(a) else 0.0) for k, (a, b) in enumerate(zip(outs, refs))]
            print('per-chunk (index, samples, rmse):', [(k, n_, f'{e_:.1e}') for k, n_, e_ in per if e_ > 1e-5])
        assert rmse < 1e-3
        engine.session_destroy(sid)
    engine.set_precision('fp16')


def test_pipelined_submit_collect_equals_sequential(engine, small_models):
    """Keeping several chunks in flight (encode | convert | decode overlapped on three streams) must not change a
    single sample: compare submit/collect at depth 4 with the oracle stream, fp32 mode."""
    from realtime_yukarin_b200.engine import SessionConfig
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    engine.set_precision('fp32')
    T, extra = 0.3, (0.0, 0.5, 0.0)
    cfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                        buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                        threshold_db=60.0, vocoder_buffer_size=1024)
    sid = engine.session_create(cfg)
    orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
    x = _speech(3.6, 44)
    n = round(T * 24000)
    nchunks = len(x) // n
    buf = np.empty(32768)
    tickets, outs = [], []
    for k in range(nchunks):
        tickets.append(engine.session_submit(sid, x[k * n:(k + 1) * n]))
        if len(tickets) > 4:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    while tickets:
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    refs = [orc.push(x[k * n:(k + 1) * n]) for k in range(nchunks)]
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse = float(np.sqrt(np.mean((y - r) ** 2)))
    print(f'pipelined depth 4: {len(y)} samples rmse {rmse:.3e}')
    assert rmse < 1e-3
    engine.session_destroy(sid)
    engine.set_precision('fp16')


def test_session_create_destroy_frees_device_memory(engine, small_models):
    """A destroyed session returns everything it allocated (buffers, analysis plans, U-Net plans, graphs): creating and
    destroying sessions on one engine, with a chunk pushed through each, must not grow the device memory in use."""
    import torch
    from realtime_yukarin_b200.engine import SessionConfig
    _load(engine, small_models)
    T = 0.3
    cfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                        buffer_time=T, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0,
                        threshold_db=60.0, vocoder_buffer_size=1024)
    chunk = _speech(1.0, 5)[:round(T * 24000)]
    free = {}
    for cycle in range(1, 51):
        sid = engine.session_create(cfg)
        engine.session_push(sid, chunk)
        engine.session_destroy(sid)
        if cycle in (5, 50):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[5] - free[50]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 45 session create / push / destroy cycles')
    assert abs(grown) < 4.0


def test_group_batched_stage2_matches_oracle_streams(engine, small_models):
    """BASELINE config 5 shape: several streams on one GPU share ONE batched stage-2 forward per step (ryk_group_*).
    Each member must still reproduce the oracle's chunked stream for ITS audio (fp32), with chunks kept in flight,
    and the fp16 (wgmma) group must stay within the end-to-end tolerance."""
    from realtime_yukarin_b200.engine import SessionConfig
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    T, extra, B = 0.3, (0.0, 0.5, 0.0), 3
    cfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                        buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                        threshold_db=60.0, vocoder_buffer_size=1024)
    n = round(T * 24000)
    xs = [_speech(2.4, 70 + i) for i in range(B)]
    xs[1] = xs[1] * np.concatenate([np.zeros(12000), np.ones(len(xs[1]) - 12000)]).astype(np.float32)   # a stream that starts silent
    nchunks = len(xs[0]) // n
    refs = []
    for i in range(B):
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        refs.append([orc.push(xs[i][k * n:(k + 1) * n]) for k in range(nchunks)])
    for precision, tol in (('fp32', 1e-3), ('fp16', 1e-3)):
        engine.set_precision(precision)
        sids = [engine.session_create(cfg) for _ in range(B)]
        gid = engine.group_create(sids)
        assert engine.group_size(gid) == B
        with pytest.raises(Exception):
            engine.session_push(sids[0], xs[0][:n])            # members are driven through the group only
        bufs = [[np.empty(32768) for _ in range(B)] for _ in range(8)]
        tickets, outs = [], [[] for _ in range(B)]

        def collect():
            t = tickets.pop(0)
            for i, o in enumerate(engine.group_collect(gid, t, bufs[t % 8])):
                outs[i].append(o.copy())
        for k in range(nchunks):
            tickets.append(engine.group_submit(gid, [x[k * n:(k + 1) * n] for x in xs]))
            if len(tickets) > 3:
                collect()
        while tickets:
            collect()
        for i in range(B):
            assert [len(o) for o in outs[i]] == [len(r) for r in refs[i]], i
            y, r = np.concatenate(outs[i]), np.concatenate(refs[i])
            rmse = float(np.sqrt(np.mean((y - r) ** 2)))
            print(f'group {precision} member {i}: {len(y)} samples rmse {rmse:.3e} signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
            assert rmse < tol
        engine.group_destroy(gid)
        for sid in sids:
            engine.session_destroy(sid)
    engine.set_precision('fp16')
