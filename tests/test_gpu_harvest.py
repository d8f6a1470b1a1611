"""Harvest f0 on the H100 (csrc/world_harvest.cu, ryk_engine_set_f0_method) against the oracle's Harvest restatement, stage by stage:
decimated waveform, raw per-channel candidates, refined candidates / scores, tracked contour, smoothed 1 ms contour, 5 ms output, then
Harvest + StoneMask through ryk_world_f0 / ryk_world_analyze and a device session in Harvest mode against the oracle stream."""
import dataclasses

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import synthetic

from .test_gpu_parity import CFG, _load, _speech

pytestmark = pytest.mark.gpu


@pytest.fixture()
def harvest_engine(engine):
    engine.set_f0_method('harvest')
    yield engine
    engine.set_f0_method('dio')


def _stage(name, got, ref, rtol, report, zero_pattern=True):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    ok = got.shape == ref.shape
    pat = bool(ok and np.array_equal(got != 0, ref != 0)) if zero_pattern else True
    err = float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-300) * (ref != 0))) if ok and got.size else 0.0
    absd = float(np.max(np.abs(got - ref))) if ok and got.size else 0.0
    good = ok and pat and (err <= rtol or absd <= 1e-12)
    report.append((name, good, f'{name}: shape {got.shape} zero-pattern {"same" if pat else "DIFFERS"} max rel {err:.2e} max abs {absd:.2e}'
                         + ('' if pat or not ok else f' ({int(((got != 0) != (ref != 0)).sum())} entries)')))
    return good


@pytest.mark.parametrize('seconds,stream', [(0.3, 4), (1.0, 7), (0.3, 33)])
def test_harvest_matches_oracle_stage_by_stage(harvest_engine, seconds, stream):
    eng = harvest_engine
    x = _speech(seconds + 0.5, stream)[: int(round(seconds * CFG.fs))]
    f0_ref, t_ref, d = oworld.harvest(x, CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil, debug=True)
    f0_sm_ref = oworld.stonemask(x.astype(np.float64), CFG.fs, t_ref, f0_ref)
    f0, t = eng.world_f0(x, CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil)
    g = eng.debug_harvest(len(x), CFG.fs, CFG.frame_period, CFG.f0_floor, CFG.f0_ceil)
    rep = []
    _stage('decimated y', g['y'], d['y'], 1e-9, rep, zero_pattern=False)
    _stage('raw candidates', g['raw'], d['raw'], 1e-9, rep)
    rep.append(('nc', g['nc'] == d['nc'], f'candidate columns {g["nc"]} vs oracle {d["nc"]}'))
    _stage('refined candidates', g['cand'], d['cand'], 1e-7, rep)
    _stage('candidate scores', g['score'], d['score'], 1e-5, rep)
    _stage('tracked contour (FixF0Contour)', g['best'], d['best'], 1e-7, rep)
    _stage('smoothed 1 ms contour', g['basic'], d['basic'], 1e-7, rep)
    _stage('harvest f0 (5 ms)', g['f0_raw'], f0_ref, 1e-7, rep)
    _stage('harvest + stonemask', f0, f0_sm_ref, 1e-7, rep)
    for _, _, line in rep:
        print(line)
    bad = [name for name, good, _ in rep if not good]
    assert not bad, f'stages differing from the oracle: {bad}'
    assert np.allclose(t, t_ref)


def test_world_analyze_in_harvest_mode(harvest_engine):
    eng = harvest_engine
    cfg = dataclasses.replace(CFG, f0_method='harvest')
    x = _speech(1.0, 5)
    ref = opipe.extract_features(x, cfg)
    out = eng.world_analyze(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length, cfg.order, cfg.alpha)
    assert np.array_equal(out['voiced'], ref['voiced'].ravel())
    assert np.allclose(out['f0'], ref['f0'].ravel(), rtol=1e-6)
    assert np.allclose(np.log(out['sp']), np.log(ref['sp']), atol=2e-4)
    assert np.allclose(out['ap'], ref['ap'], atol=1e-5)
    # and the extractor really changed: DIO's contour differs from Harvest's
    eng.set_f0_method('dio')
    dio = eng.world_analyze(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length, cfg.order, cfg.alpha)
    eng.set_f0_method('harvest')
    assert not np.array_equal(dio['f0'], out['f0'])


def test_session_in_harvest_mode_matches_oracle_stream(harvest_engine, small_models):
    """Harvest inside the pipelined session's analysis graph (0.3 s chunks, FP32 convs) == the oracle's chunked stream in Harvest mode."""
    from realtime_yukarin_b200.engine import SessionConfig
    eng = harvest_engine
    ac, sr, f0c = _load(eng, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    eng.set_precision('fp32')
    try:
        T, extra = 0.3, (0.0, 0.5, 0.0)
        scfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                             buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                             threshold_db=60.0, vocoder_buffer_size=1024)
        sid = eng.session_create(scfg)
        orc = opipe.StreamOracle(dataclasses.replace(CFG, f0_method='harvest'), p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        x = _speech(2.4, 33)
        n = round(T * 24000)
        outs, refs = [], []
        for k in range(len(x) // n):
            y = eng.session_push(sid, x[k * n:(k + 1) * n])
            r = orc.push(x[k * n:(k + 1) * n])
            assert len(y) == len(r), (k, len(y), len(r))
            outs.append(y.copy()); refs.append(r)
        y, r = np.concatenate(outs), np.concatenate(refs)
        rmse = float(np.sqrt(np.mean((y - r) ** 2)))
        print(f'harvest session: {len(y)} samples, rmse {rmse:.3e}, signal rms {float(np.sqrt(np.mean(r ** 2))):.3e}')
        assert rmse < 1e-3
        eng.session_destroy(sid)
    finally:
        eng.set_precision('fp16')
