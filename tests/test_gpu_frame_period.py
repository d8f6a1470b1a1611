"""Frame periods other than 5 ms on the H100, against the oracle at the same period.

Every kernel of the analysis and synthesis path takes the frame period at run time: DIO's candidate times and FixF0Contour window
(3 frames at 10 ms, 29 at 1 ms), the frame centres of StoneMask, CheapTrick and D4C, Harvest's subsampling of its 1 ms contour, the
synthesizers' frame times and interpolation, and the session's hop, frame counts, windows and output capacity.  Each case below asserts
what the 5 ms test of the same path asserts, at the same tolerance, over 1, 2, 4, 8 and 10 ms with 5 ms in the same parametrization as
the control; each prints its errors, so that the other periods can be read against the control's level, not only against the bound.

  a. WORLD analysis (tests/test_gpu_parity.py): world_analyze and world_f0 on speech, on a glide through f0_floor, and on a signal
     whose f0_length is vrm + 2 at 1 ms, and on the shortest start of a voice in which DIO keeps a voiced frame at 1 ms;
  b. Harvest stage by stage (tests/test_gpu_harvest.py) and world_analyze in Harvest mode, at 1, 4 and 10 ms;
  c. offline synthesis (tests/test_gpu_widen.py) and the realtime synthesizer in 60-frame pieces, with vocoder blocks of 256 to 2048
     samples at 5 and 10 ms (tests/test_gpu_parity.py);
  d. FP32 sessions with base-16 models through submit / collect at depth 4 against StreamOracle, their io geometry against
     tests/session_geometry.py; one FP16 base-64 session at 10 ms under the headline bounds (tests/test_gpu_headline_parity.py), one
     Harvest session at 4 ms, and one CREPE session at a 10 ms step against the host chain (tests/test_gpu_crepe_session.py);
  e. periods that do not divide 1000 ms are refused at creation, allocating and launching nothing;
  f. RealtimePipeline runs at the models' frame period when Config says another, and its snapshots check that period.
"""
import dataclasses

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import SessionConfig

from .test_frame_period_oracle import (PERIODS, PIDS, acoustic_param, geometry, glide, oracle_pipeline_stream, pipeline_config,
                                       short_signal, vrm, write_models_at)
from .test_gpu_harvest import _stage
from .test_gpu_headline_parity import _waveform_spectral_distance
from .test_gpu_parity import _load, _speech

pytestmark = pytest.mark.gpu

FS = 24000


def _signal(name):
    if name == 'speech':
        return _speech(0.6, 1)
    if name == 'glide':
        return glide(0.5, stream=1)
    return short_signal(name)


@pytest.fixture(scope='module')
def models_10ms(tmp_path_factory):
    """base-16 models whose configuration says 10 ms"""
    return write_models_at(tmp_path_factory.mktemp('models_10ms'), 10)


@pytest.fixture
def fp32(engine):
    engine.set_precision('fp32')
    yield engine
    engine.set_precision('fp16')


# ---- a. WORLD analysis ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
@pytest.mark.parametrize('signal', ['speech', 'glide', 'short', 'edge'])
def test_world_analysis_matches_oracle(engine, fp, signal):
    cfg = opipe.PathConfig(frame_period=fp)
    x = _signal(signal)
    ref = opipe.extract_features(x, cfg)
    got = engine.world_analyze(x, cfg.fs, fp, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length, cfg.order, cfg.alpha)
    f0r, f0g = ref['f0'].ravel().astype(np.float64), got['f0'].astype(np.float64)
    assert len(f0g) == len(f0r) == len(x) // cfg.hop
    e_f0 = float(np.max(np.abs(f0g - f0r) / np.maximum(f0r, 1e-300) * (f0r != 0))) if len(f0r) else 0.0
    e_sp = float(np.abs(np.log(got['sp']) - np.log(ref['sp'])).max())
    e_ap, e_mc = float(np.abs(got['ap'] - ref['ap']).max()), float(np.abs(got['mc'] - ref['mc']).max())
    # f0 in double precision through world_f0
    f0_ref, t = oworld.dio(x.astype(np.float64), cfg.fs, fp, cfg.f0_floor, cfg.f0_ceil)
    f0_ref = oworld.stonemask(x.astype(np.float64), cfg.fs, t, f0_ref)
    f0, tt = engine.world_f0(x, cfg.fs, fp, cfg.f0_floor, cfg.f0_ceil)
    e_f64 = float(np.max(np.abs(f0 - f0_ref) / np.maximum(f0_ref, 1e-300) * (f0_ref != 0)))
    print(f'{fp:g} ms {signal}: {len(f0r)} frames ({int((f0r > 0).sum())} voiced, lowest {f0r[f0r > 0].min() if (f0r > 0).any() else 0:.1f} Hz), '
          f'vrm {vrm(fp)}; f0 rel {e_f0:.1e}, f0 fp64 rel {e_f64:.1e}, log sp {e_sp:.1e}, ap {e_ap:.1e}, mc {e_mc:.1e}')
    assert np.array_equal(f0r != 0, f0g != 0)
    assert np.allclose(f0g, f0r, rtol=1e-6, atol=0)
    assert np.array_equal(ref['voiced'].ravel(), got['voiced'])
    assert np.allclose(np.log(got['sp']), np.log(ref['sp']), atol=2e-4)
    assert np.allclose(got['ap'], ref['ap'], rtol=1e-4, atol=1e-6)
    assert np.allclose(got['mc'], ref['mc'], atol=2e-4)
    assert len(f0) == len(f0_ref) and np.array_equal(f0 != 0, f0_ref != 0)
    assert np.allclose(f0, f0_ref, rtol=1e-9)
    assert np.allclose(tt, t)


# ---- b. Harvest -----------------------------------------------------------------------------------------------------------------
@pytest.fixture
def harvest(engine):
    engine.set_f0_method('harvest')
    yield engine
    engine.set_f0_method('dio')


@pytest.mark.parametrize('fp', [1.0, 4.0, 5.0, 10.0], ids=['1ms', '4ms', '5ms', '10ms'])
def test_harvest_matches_oracle_stage_by_stage(harvest, fp):
    x = _speech(0.6, 7)
    f0_ref, t_ref, d = oworld.harvest(x, FS, fp, 71.0, 800.0, debug=True)
    f0_sm_ref = oworld.stonemask(x.astype(np.float64), FS, t_ref, f0_ref)
    f0, t = harvest.world_f0(x, FS, fp, 71.0, 800.0)
    g = harvest.debug_harvest(len(x), FS, fp, 71.0, 800.0)
    rep = []
    _stage('decimated y', g['y'], d['y'], 1e-9, rep, zero_pattern=False)
    _stage('raw candidates', g['raw'], d['raw'], 1e-9, rep)
    rep.append(('nc', g['nc'] == d['nc'], f'candidate columns {g["nc"]} vs oracle {d["nc"]}'))
    _stage('refined candidates', g['cand'], d['cand'], 1e-7, rep)
    _stage('candidate scores', g['score'], d['score'], 1e-5, rep)
    _stage('tracked contour (FixF0Contour)', g['best'], d['best'], 1e-7, rep)
    _stage('smoothed 1 ms contour', g['basic'], d['basic'], 1e-7, rep)
    _stage(f'harvest f0 ({fp:g} ms)', g['f0_raw'], f0_ref, 1e-7, rep)
    _stage('harvest + stonemask', f0, f0_sm_ref, 1e-7, rep)
    for _, _, line in rep:
        print(f'{fp:g} ms {line}')
    bad = [name for name, good, _ in rep if not good]
    assert not bad, f'stages differing from the oracle: {bad}'
    assert np.allclose(t, t_ref)
    # world_analyze in Harvest mode
    cfg = opipe.PathConfig(frame_period=fp, f0_method='harvest')
    ref = opipe.extract_features(x, cfg)
    out = harvest.world_analyze(x, FS, fp, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length, cfg.order, cfg.alpha)
    print(f'{fp:g} ms harvest world_analyze: f0 max rel {float(np.max(np.abs(out["f0"] - ref["f0"].ravel()) / np.maximum(ref["f0"].ravel(), 1e-300))):.1e}, '
          f'log sp {float(np.abs(np.log(out["sp"]) - np.log(ref["sp"])).max()):.1e}, ap {float(np.abs(out["ap"] - ref["ap"]).max()):.1e}')
    assert np.array_equal(out['voiced'], ref['voiced'].ravel())
    assert np.allclose(out['f0'], ref['f0'].ravel(), rtol=1e-6)
    assert np.allclose(np.log(out['sp']), np.log(ref['sp']), atol=2e-4)
    assert np.allclose(out['ap'], ref['ap'], atol=1e-5)


# ---- c. synthesis ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
def test_offline_synthesis_matches_oracle(engine, fp):
    x = synthetic.synthetic_speech(1.0, stream=2)
    f = opipe.extract_features(x, opipe.PathConfig(frame_period=fp))
    f0 = f['f0'].ravel().astype(np.float64)
    yr, ir, sr_, vr = oworld.synthesize(f0, f['sp'], f['ap'], FS, fp, return_pulses=True)
    yg, ig, sg_, vg = engine.world_synthesize(f0, f['sp'], f['ap'], FS, fp, return_pulses=True)
    assert len(yg) == len(yr) == int(len(f0) * fp * FS / 1000)
    assert np.array_equal(ig, ir), 'pulse positions differ'
    assert np.array_equal(vg, vr), 'voiced flags at the pulses differ'
    rmse = float(np.sqrt(np.mean((yg - yr) ** 2)))
    print(f'{fp:g} ms offline synthesis: {len(f0)} frames, {len(ir)} pulses, shift max err {float(np.abs(sg_ - sr_).max()):.1e}, '
          f'rmse {rmse:.3e} (peak {float(np.abs(yr).max()):.3f})')
    assert np.allclose(sg_, sr_, rtol=0, atol=1e-12)
    assert rmse <= 1e-9 * max(1.0, float(np.abs(yr).max()))


SYNTH_CASES = [(fp, 1024) for fp in PERIODS] + [(fp, b) for fp in (5.0, 10.0) for b in (256, 512, 2048)]


@pytest.mark.parametrize('fp,block', SYNTH_CASES, ids=[f'{fp:g}ms-{b}' for fp, b in SYNTH_CASES])
def test_realtime_synthesizer_matches_oracle(engine, fp, block):
    x = _speech(1.2, 7)
    f = opipe.extract_features(x, opipe.PathConfig(frame_period=fp))
    fft = oworld.cheaptrick_fft_size(FS)
    ref_s = oworld.RealtimeSynthesizer(FS, fp, fft, block)
    sid = engine.synth_create(FS, fp, fft, block)
    total_ref, total_got = [], []
    try:
        for a in range(0, len(f['f0']), 60):
            sl = slice(a, a + 60)
            f0 = f['f0'][sl].ravel().astype(np.float64)
            yr = ref_s.decode(f0, f['sp'][sl], f['ap'][sl])
            yg = engine.synth_decode(sid, f0, f['sp'][sl], f['ap'][sl])
            assert len(yr) == len(yg), (a, len(yr), len(yg))
            total_ref.append(yr)
            total_got.append(yg)
    finally:
        engine.synth_destroy(sid)
    yr, yg = np.concatenate(total_ref), np.concatenate(total_got)
    assert len(yr) >= 4 * block and len(yr) % block == 0
    rmse = float(np.sqrt(np.mean((yr - yg) ** 2)))
    print(f'{fp:g} ms block {block}: {len(f["f0"])} frames, {len(yr)} samples, synth rmse {rmse:.3e}, rms {float(np.sqrt(np.mean(yr ** 2))):.3e}')
    assert rmse < 1e-6 * max(1.0, float(np.abs(yr).max()) * 1e3)


# ---- d. sessions ----------------------------------------------------------------------------------------------------------------
def _session_cfg(geo, block=1024):
    return geo.session_config(60.0, block=block)


def _submit_collect(engine, sid, chunks, depth):
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    tickets, outs = [], []
    for c in chunks:
        tickets.append(engine.session_submit(sid, c))
        if len(tickets) > depth:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    while tickets:
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    return outs


def _oracle_stream(paths, cfg, geo, stats, chunks):
    p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
    orc = opipe.StreamOracle(cfg, p1, p2, stats, buffer_time=geo.buffer_time, extra=geo.extra, backend='torch')
    return [orc.push(c) for c in chunks]


def _chunks(x, geo, steps):
    assert len(x) >= steps * geo.n_wave
    return [np.ascontiguousarray(x[k * geo.n_wave:(k + 1) * geo.n_wave], np.float32) for k in range(steps)]


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
@pytest.mark.parametrize('extras', ['conv', 'all'])
def test_fp32_session_matches_oracle_stream(engine, small_models, fp32, fp, extras):
    """12 chunks through submit / collect with 4 in flight against StreamOracle at the same period: sample RMSE <= 1e-3"""
    _, _, f0c = _load(engine, small_models)
    engine.set_precision('fp32')
    geo = geometry(fp, extras)
    steps = 12
    chunks = _chunks(_speech((steps + 1) * geo.buffer_time, 33), geo, steps)
    sid = engine.session_create(_session_cfg(geo))
    try:
        g = engine.session_io_geometry(sid)
        assert (g['n_in'], g['max_out']) == (geo.n_wave, geo.max_out(1024))
        outs = _submit_collect(engine, sid, chunks, 4)
    finally:
        engine.session_destroy(sid)
    refs = _oracle_stream(small_models, opipe.PathConfig(frame_period=fp), geo, f0c.stats(), chunks)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse, rms = float(np.sqrt(np.mean((y - r) ** 2))), float(np.sqrt(np.mean(r ** 2)))
    print(f'{fp:g} ms session {geo.buffer_time} s extra {geo.extra}: n_feat {geo.n_feat} Tw {geo.Tw} Td {geo.Td}, {len(y)} samples, '
          f'rmse {rmse:.3e}, signal rms {rms:.3e}')
    assert rms > 1e-2
    assert rmse < 1e-3


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
def test_session_io_geometry_follows_period_and_block(engine, small_models, fp):
    _load(engine, small_models)
    for extras in ('conv', 'all'):
        geo = geometry(fp, extras)
        for block in (256, 512, 1024, 2048):
            sid = engine.session_create(_session_cfg(geo, block))
            g = engine.session_io_geometry(sid)
            engine.session_destroy(sid)
            assert (g['n_in'], g['max_out'], g['in_rate'], g['out_rate']) == (geo.n_wave, geo.max_out(block), FS, FS), (extras, block, g)


def test_fp16_full_model_session_at_10ms(engine, full_models):
    """the headline configuration (0.3 s, extras (0, 0.5, 0), 12 chunks, 3 in flight, base 64, FP16) at 10 ms, on the input
    tests/test_gpu_headline_parity.py streams at 5 ms: sample RMSE <= 1e-3, per-frame log-STFT distance <= 0.1"""
    _, _, f0c = _load(engine, full_models)
    engine.set_precision('fp16')
    geo = geometry(10.0, 'conv')
    steps = 12
    chunks = _chunks(synthetic.synthetic_speech((steps + 1) * geo.buffer_time, stream=91), geo, steps)
    sid = engine.session_create(_session_cfg(geo))
    try:
        outs = _submit_collect(engine, sid, chunks, 3)
    finally:
        engine.session_destroy(sid)
    refs = _oracle_stream(full_models, opipe.PathConfig(frame_period=10.0), geo, f0c.stats(), chunks)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse, rms = float(np.sqrt(np.mean((y - r) ** 2))), float(np.sqrt(np.mean(r ** 2)))
    lsd = _waveform_spectral_distance(y, r)
    print(f'10 ms fp16 base-64 session: {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), log-STFT distance {lsd:.3e}')
    assert rms > 1e-2
    assert rmse <= 1e-3
    assert lsd <= 0.1


def test_harvest_session_at_4ms(engine, small_models, fp32, harvest):
    _, _, f0c = _load(engine, small_models)
    engine.set_precision('fp32')
    geo = geometry(4.0, 'conv')
    steps = 10
    chunks = _chunks(_speech((steps + 1) * geo.buffer_time, 33), geo, steps)
    sid = engine.session_create(_session_cfg(geo))
    try:
        outs = [engine.session_push(sid, c).copy() for c in chunks]
    finally:
        engine.session_destroy(sid)
    refs = _oracle_stream(small_models, opipe.PathConfig(frame_period=4.0, f0_method='harvest'), geo, f0c.stats(), chunks)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse = float(np.sqrt(np.mean((y - r) ** 2)))
    print(f'4 ms harvest session: {len(y)} samples, rmse {rmse:.3e}, signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
    assert rmse < 1e-3


def test_crepe_session_at_10ms_matches_host_chain(engine, models_10ms, fp32, tmp_path):
    """CREPE at a 10 ms step: the session against EncodeStream / ConvertStream / DecodeStream with Vocoder(extract_f0_mode=CREPE) built
    from models whose acoustic_param says 10 ms; sample RMSE < 1e-3"""
    from realtime_yukarin_b200 import crepe as pcrepe
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.stream import ConvertStream, DecodeStream, EncodeStream, StreamWrapper
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    ac, sr, _ = _load(engine, models_10ms)
    pcrepe.load_crepe_model(synthetic.write_crepe_model(tmp_path, seed=5, capacity='tiny'), engine)
    acp = acoustic_param(models_10ms)
    assert acp.frame_period == 10
    engine.set_precision('fp32')
    T, extra = 0.3, (0.0, 0.5, 0.0)
    voc = RealtimeVocoder(acoustic_param=acp, out_sampling_rate=FS, extract_f0_mode=VocodeMode.CREPE)
    voc.create_synthesizer(buffer_size=1024, number_of_pointers=16)
    es, cs, ds = EncodeStream(voc), ConvertStream(VoiceChanger(ac, sr, threshold=60)), DecodeStream(voc)
    ws = [StreamWrapper(es, extra[0]), StreamWrapper(cs, extra[1]), StreamWrapper(ds, extra[2])]
    x = _speech(2.4, 52)
    n = round(T * FS)
    refs = []
    for k in range(len(x) // n):
        es.add(start_time=extra[0] + k * T, data=x[k * n:(k + 1) * n])
        cs.add(start_time=extra[1] + k * T, data=ws[0].process_next(T))
        ds.add(start_time=extra[2] + k * T, data=ws[1].process_next(T))
        refs.append(ws[2].process_next(T))
    geo = geometry(10.0, 'conv')
    engine.set_f0_method('crepe')
    try:
        sid = engine.session_create(_session_cfg(geo))
    finally:
        engine.set_f0_method('dio')
    try:
        outs = [engine.session_push(sid, x[k * n:(k + 1) * n]).copy() for k in range(len(x) // n)]
    finally:
        engine.session_destroy(sid)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    rmse = float(np.sqrt(np.mean((y - r) ** 2)))
    print(f'10 ms crepe session: {len(y)} samples, rmse {rmse:.3e}, signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
    assert len(y) > 0 and rmse < 1e-3


# ---- e. refusals ----------------------------------------------------------------------------------------------------------------
# chunks of whole frames at each period (0.3 s is 100 frames of 3 ms, 50 of 6 ms; 0.294 s 42 of 7 ms; 0.306 s 34 of 9 ms), so that
# only the period itself is wrong
REFUSED = [(3.0, 0.3), (6.0, 0.3), (7.0, 0.294), (9.0, 0.306)]


def test_periods_that_do_not_divide_a_second_are_refused(engine, small_models):
    import torch
    from realtime_yukarin_b200.engine import RykError
    from realtime_yukarin_b200.worker import RealtimePipeline
    _load(engine, small_models)
    engine.synchronize()
    free, before = torch.cuda.mem_get_info()[0], engine.launch_count
    for _ in range(5):
        for fp, bt in REFUSED:
            cfg = SessionConfig(fs=FS, frame_period_ms=fp, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                                buffer_time=bt, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0, threshold_db=60.0,
                                vocoder_buffer_size=1024)
            with pytest.raises(RykError, match='frame period must divide 1000 ms'):
                engine.session_create(cfg)
    engine.synchronize()
    assert engine.launch_count == before
    assert abs(torch.cuda.mem_get_info()[0] - free) < 2**20, (free, torch.cuda.mem_get_info()[0])
    # a pipeline built from a model at such a period gets the session's refusal
    config = pipeline_config(small_models, frame_period=5.0, buffer_time=0.3)
    with pytest.raises(RykError, match='frame period must divide 1000 ms'):
        RealtimePipeline(config, acoustic_param=dataclasses.replace(acoustic_param(small_models), frame_period=6), engine=engine)


# ---- f. the pipeline at the models' period --------------------------------------------------------------------------------------
def test_pipeline_runs_at_the_models_frame_period(engine, models_10ms, fp32):
    """models at 10 ms and a Config that says 5 ms: RealtimePipeline plays the 10 ms oracle stream (sample RMSE <= 1e-3, the same silent
    chunks); its snapshot restores with the models' parameters and is refused at the 5 ms a missing model implies"""
    from realtime_yukarin_b200.worker import RealtimePipeline
    _, _, f0c = _load(engine, models_10ms)
    engine.set_precision('fp32')
    acp = acoustic_param(models_10ms)
    config = pipeline_config(models_10ms, frame_period=5.0)
    x = synthetic.synthetic_speech(3.3, stream=17)
    n = config.in_audio_chunk
    pipe = RealtimePipeline(config, acoustic_param=acp, engine=engine, depth=2)
    try:
        assert engine.session_io_geometry(pipe._sid)['max_out'] == geometry(10.0, 'conv').max_out(1024)
        got = [pipe.process(x[k * n:(k + 1) * n], block=True) for k in range(len(x) // n)]
        assert pipe.drain() == []
        blob = pipe.snapshot()
    finally:
        pipe.close()
    want = oracle_pipeline_stream(models_10ms, config, 10.0, x, f0c.stats())
    assert sum(w.any() for w in want) >= 4
    assert [g.any() for g in got] == [w.any() for w in want]
    rmse = float(np.sqrt(np.mean((np.concatenate(got) - np.concatenate(want)) ** 2)))
    at_5ms = oracle_pipeline_stream(models_10ms, config, 5.0, x, f0c.stats())
    off = float(np.sqrt(np.mean((np.concatenate(got) - np.concatenate(at_5ms)) ** 2)))
    print(f'pipeline with 10 ms models, Config 5 ms: {len(got)} chunks, rmse {rmse:.3e} against the 10 ms oracle stream, '
          f'{off:.3e} against the 5 ms one')
    assert rmse <= 1e-3
    dst = RealtimePipeline.restore(blob, config, engine=engine, acoustic_param=acp)
    dst.close()
    with pytest.raises(ValueError, match='model frame_period: recorded 10.0, config 5.0'):
        RealtimePipeline.restore(blob, config, engine=engine)
