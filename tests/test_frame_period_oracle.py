"""Frame periods other than 5 ms, on the CPU.

Every stage of the analysis and synthesis path takes the frame period at run time and derives frame times, window widths and
capacities from it (DIO's FixF0Contour window is 2 * round(1000 / fp / f0_floor) + 1 frames: 3 at 10 ms, 29 at 1 ms).  Here:
  a. the oracle's DIO, StoneMask, CheapTrick, D4C and realtime synthesizer agree with the independent numpy writings of
     tests/independent_world.py at every period that divides 1000 ms, at the tolerances tests/test_oracle.py holds them to at 5 ms,
     so that a GPU mismatch at such a period (tests/test_gpu_frame_period.py) is the kernel's;
  b. RealtimePipeline runs at the stage-1 model's acoustic_param.frame_period, not at Config.frame_period (which the reference reads
     and never uses), and restoring a pipeline snapshot checks the model's period;
  c. tests/session_geometry.py's shapes follow the frame period as the oracle stream and the pipeline size them.
"""
import json

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as W
from realtime_yukarin_b200 import synthetic

from . import independent_world as iw
from . import session_geometry as sg
from .fake_engine import OracleEngine

FS = 24000
PERIODS = [1.0, 2.0, 4.0, 5.0, 8.0, 10.0]          # the whole-millisecond periods that divide 1000 ms
PIDS = [f'{p:g}ms' for p in PERIODS]
STATS = (float(np.log(150.0)), 0.2, float(np.log(250.0)), 0.2)


def vrm(frame_period, f0_floor=71.0):
    """frames of DIO's FixF0Contour window at this period"""
    return int(0.5 + 1000.0 / frame_period / f0_floor) * 2 + 1


def glide(seconds, stream=0, f_hi=190.0, f_lo=62.0):
    """a harmonic voice whose f0 falls exponentially from f_hi to f_lo, through f0_floor (71 Hz), then rises back: the contour DIO
    repairs near the floor; -40 dB noise"""
    rng = np.random.default_rng(500 + stream)
    n = int(round(seconds * FS))
    u = np.abs(np.linspace(-1.0, 1.0, n))
    f0 = f_lo * (f_hi / f_lo) ** u
    phase = 2 * np.pi * np.cumsum(f0) / FS
    x = sum(np.sin(h * phase + rng.uniform(0, 2 * np.pi)) / h for h in range(1, 16))
    x = 0.2 * x / np.abs(x).max() + 1e-3 * rng.standard_normal(n)
    return x.astype(np.float32)


def write_models_at(directory, frame_period, seed=3, base1=16, base2=16):
    """synthetic model files whose configuration says `frame_period` (the weights do not depend on it)"""
    paths = synthetic.write_synthetic_models(directory, seed=seed, base1=base1, base2=base2)
    c = json.loads(paths['stage1_config_path'].read_text())
    c['dataset']['acoustic_param']['frame_period'] = int(frame_period)
    paths['stage1_config_path'].write_text(json.dumps(c, indent=1))
    c = json.loads(paths['stage2_config_path'].read_text())
    c['dataset']['param']['acoustic_feature_param']['frame_period'] = int(frame_period)
    paths['stage2_config_path'].write_text(json.dumps(c, indent=1))
    return paths


def acoustic_param(paths):
    from realtime_yukarin_b200.params import create_from_json
    return create_from_json(paths['stage1_config_path']).dataset.acoustic_param


def pipeline_config(paths, frame_period=5.0, **kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=24000, output_rate=24000, frame_period=frame_period,
                  buffer_time=0.3, extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=0.5, output_scale=2.0,
                  input_silent_threshold=60.0, output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5,
                  decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: paths[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                     'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


# ---- a. the oracle against the independent writings ----------------------------------------------------------------------------
def test_glide_reaches_the_f0_floor():
    x = glide(0.6).astype(np.float64)
    f0, t = W.dio(x, FS, 5.0)[:2]
    f0 = W.stonemask(x, FS, t, f0)
    assert 0 < f0[f0 > 0].min() < 80.0 and (f0 > 0).sum() > 60


def short_signal(name):
    """'short': f0_length vrm + 2 = 31 frames at 1 ms; 'edge': 88 frames at 1 ms, the shortest start of this voice in which DIO keeps a
    voiced frame (one, at frame 44; 87 frames keep none, 89 keep 88)"""
    x = synthetic.synthetic_speech(1.0, stream=1)
    return x[:(vrm(1.0) + 1) * 24] if name == 'short' else x[:87 * 24]


SIGNALS = {'speech': lambda: synthetic.synthetic_speech(0.5, stream=9), 'glide': lambda: glide(0.5, stream=1),
           'short': lambda: short_signal('short'), 'edge': lambda: short_signal('edge')}


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
@pytest.mark.parametrize('signal', list(SIGNALS))
def test_dio_and_stonemask_agree_with_independent_numpy_writings(fp, signal):
    """same frame times and voiced decisions, f0 within 1e-9 Hz"""
    x = SIGNALS[signal]().astype(np.float64)
    f0_ref, t_ref = W.dio(x, FS, fp)[:2]
    f0, t = iw.dio_np(x, FS, fp)
    assert len(t_ref) == int(1000.0 * len(x) / FS / fp) + 1
    if fp == 1.0 and signal in ('short', 'edge'):
        assert (len(t_ref), int((f0_ref > 0).sum())) == ((vrm(fp) + 2, 0) if signal == 'short' else (88, 1))
    assert np.array_equal(t, t_ref) and np.array_equal(f0 > 0, f0_ref > 0)
    if signal in ('speech', 'glide'):
        assert (f0_ref > 0).sum() > 0.3 * len(f0_ref)
    assert np.abs(f0 - f0_ref).max() < 1e-9
    assert np.abs(iw.stonemask_np(x, FS, t_ref, f0_ref) - W.stonemask(x, FS, t_ref, f0_ref)).max() < 1e-9


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
def test_cheaptrick_and_d4c_agree_with_independent_numpy_writings(fp):
    x = synthetic.synthetic_speech(0.4, stream=5).astype(np.float64)
    f0, t = W.dio(x, FS, fp)[:2]
    f0 = W.stonemask(x, FS, t, f0)
    assert (f0 > 0).sum() > 0 and (f0 == 0).sum() > 0
    sp = W.cheaptrick(x, FS, t, f0)
    assert np.abs(np.log(iw.cheaptrick_np(x, FS, t, f0)) - np.log(sp)).max() < 1e-8
    ap = W.d4c(x, FS, t, f0)
    ap = ap[0] if isinstance(ap, tuple) else ap
    assert np.abs(iw.d4c_np(x, FS, t, f0) - ap).max() < 1e-10


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
def test_realtime_synthesizer_agrees_with_an_independent_numpy_writing(fp):
    """60-frame pieces: identical pulses and block counts, samples within 1e-12"""
    x = synthetic.synthetic_speech(1.0, stream=7)
    f = opipe.extract_features(x, opipe.PathConfig(frame_period=fp))
    ref, mine = W.RealtimeSynthesizer(FS, fp, 1024, 1024), iw.NumpyRealtimeSynth(FS, fp, 1024, 1024)
    total = 0
    for a in range(0, len(f['f0']), 60):
        f0 = f['f0'][a:a + 60].ravel().astype(np.float64)
        yr, ym = ref.decode(f0, f['sp'][a:a + 60], f['ap'][a:a + 60]), mine.decode(f0, f['sp'][a:a + 60], f['ap'][a:a + 60])
        assert len(yr) == len(ym)
        if len(yr):
            assert np.abs(yr - ym).max() < 1e-12
        total += len(yr)
    idx, _, vuv = ref.pulses()
    assert total >= 8 * 1024 and len(idx) > 60
    assert np.array_equal(idx, [p[0] for p in mine.pulses]) and np.array_equal(vuv, [p[2] for p in mine.pulses])


# ---- b. the pipeline runs at the model's frame period ---------------------------------------------------------------------------
@pytest.fixture(scope='module')
def models_10ms(tmp_path_factory):
    return write_models_at(tmp_path_factory.mktemp('models_10ms'), 10)


def oracle_pipeline_stream(paths, config, fp, x, stats=STATS):
    """what RealtimePipeline.process plays for the chunks of x at frame period fp: StreamOracle + the decode worker's re-blocker"""
    p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
    orc = opipe.StreamOracle(opipe.PathConfig(frame_period=fp, threshold_db=config.input_silent_threshold), p1, p2, stats,
                             buffer_time=config.buffer_time, extra=(config.encode_extra_time, config.convert_extra_time,
                                                                    config.decode_extra_time), backend='torch')
    rb = opipe.OutputReblockOracle(config.out_audio_chunk, config.output_silent_threshold)
    n = config.in_audio_chunk
    want = []
    for k in range(len(x) // n):
        _, c = rb.push(orc.push((x[k * n:(k + 1) * n] * config.input_scale).astype(np.float32)))
        want.append(np.zeros(config.out_audio_chunk, np.float32) if c is None
                    else (c * config.output_scale)[:config.out_audio_chunk].astype(np.float32))
    return want


def test_pipeline_takes_the_frame_period_from_the_model(models_10ms):
    """models at 10 ms and a Config that says 5 ms: the pipeline's stream is the 10 ms oracle stream, not the 5 ms one"""
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = OracleEngine(models_10ms['stage1_model_path'], models_10ms['stage2_model_path'])
    fake.f0_set_stats(*STATS)
    config = pipeline_config(models_10ms, frame_period=5.0)
    acp = acoustic_param(models_10ms)
    assert acp.frame_period == 10
    x = synthetic.synthetic_speech(2.1, stream=17)
    pipe = RealtimePipeline(config, acoustic_param=acp, engine=fake, depth=2)
    assert fake.sessions[0]['orc'].cfg.frame_period == 10.0 and fake.sessions[0]['orc'].n_feat == 30
    n = config.in_audio_chunk
    got = [pipe.process(x[k * n:(k + 1) * n], block=True) for k in range(len(x) // n)]
    pipe.close()
    want = oracle_pipeline_stream(models_10ms, config, 10.0, x)
    at_5ms = oracle_pipeline_stream(models_10ms, config, 5.0, x)
    assert sum(w.any() for w in want) >= 3
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    assert not all(np.array_equal(g, w) for g, w in zip(got, at_5ms))


def _pipeline_blob(frame_period, config):
    from realtime_yukarin_b200 import snapshot
    from .test_session_snapshot import MoveEngine, _drained_pipeline, _reblock_blob, _session_conf
    conf = _session_conf()
    conf.cfg.frame_period_ms = frame_period
    sb = snapshot.pack('session', [('CONF', bytes(conf)), ('HOST', b'\x01' * 24), ('WAVE', b'\x02' * 13)])
    return _drained_pipeline(MoveEngine(sb, _reblock_blob(chunk=config.out_audio_chunk)), config).snapshot()


def test_pipeline_restore_checks_the_models_frame_period(small_models, models_10ms):
    from realtime_yukarin_b200.worker import RealtimePipeline
    from .test_session_snapshot import MoveEngine
    config = pipeline_config(models_10ms, frame_period=5.0, input_scale=1.0, output_scale=1.0, buffer_time=0.1)
    acp10, acp5 = acoustic_param(models_10ms), acoustic_param(small_models)
    blob10, blob5 = _pipeline_blob(10.0, config), _pipeline_blob(5.0, config)
    RealtimePipeline.restore(blob10, config, engine=MoveEngine(), acoustic_param=acp10)
    RealtimePipeline.restore(blob5, config, engine=MoveEngine(), acoustic_param=acp5)
    RealtimePipeline.restore(blob5, config, engine=MoveEngine())            # no model parameters: 5 ms, as the constructor takes it
    for blob, acp in ((blob10, acp5), (blob10, None), (blob5, acp10)):
        dst = MoveEngine()
        with pytest.raises(ValueError, match='another configuration: model frame_period'):
            RealtimePipeline.restore(blob, config, engine=dst, acoustic_param=acp)
        assert dst.calls == []


# ---- c. the geometry table at every frame period -------------------------------------------------------------------------------
def geometry(fp, extras):
    """0.3 s chunks (0.32 s at 8 ms, where 0.3 s is 37.5 frames) with extras (0, 0.5, 0) or, with 'all', three non-zero ones; the
    chunk and the encode extra are whole frames, as the session requires"""
    bt = 0.3 if round(300 / fp) * fp == 300 else 0.32
    return sg.Geometry(f'{extras}-{fp:g}ms', bt, (0.0, 0.5, 0.0) if extras == 'conv' else (0.04, 0.2, 0.04), frame_period=fp)


@pytest.mark.parametrize('fp', PERIODS, ids=PIDS)
@pytest.mark.parametrize('extras', ['conv', 'all'])
def test_geometry_follows_the_frame_period(small_models, extras, fp):
    """Geometry's shapes at fp == StreamOracle's windows == the host stream classes' frame rate, and max_out == the capacity the
    pipeline gives one step's output"""
    from realtime_yukarin_b200.worker import RealtimePipeline
    g = geometry(fp, extras)
    assert g.rate * fp == 1000 and g.rate == 1000 // int(fp) and g.hop == 24 * fp
    assert g.n_wave == g.n_feat * g.hop and g.e_wave == g.e_enc * g.hop
    assert g.Tw == g.n_feat + 2 * round(g.extra[1] * 1000 / fp) and g.Td == g.n_feat + 2 * round(g.extra[2] * 1000 / fp)
    assert g.Tw < g.Tp <= g.Tw + 128 and g.buckets <= sg.MAX_BUCKETS
    orc = opipe.StreamOracle(opipe.PathConfig(frame_period=fp), None, None, STATS, buffer_time=g.buffer_time, extra=g.extra)
    assert (orc.rate, orc.n_wave, orc.n_feat, orc.e_wave, orc.e_conv, orc.e_dec) == (g.rate, g.n_wave, g.n_feat, g.e_wave, g.e_conv, g.e_dec)
    assert round(g.extra[0] * orc.rate) == g.e_enc
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    config = pipeline_config(small_models, buffer_time=g.buffer_time, encode_extra_time=g.extra[0], convert_extra_time=g.extra[1],
                             decode_extra_time=g.extra[2], vocoder_buffer_size=512)
    pipe = RealtimePipeline(config, acoustic_param=type('P', (), {'frame_period': int(fp)})(), engine=fake)
    assert len(pipe._scratch) == g.max_out(512)
    pipe.close()
