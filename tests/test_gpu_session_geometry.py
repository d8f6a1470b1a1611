"""Streaming sessions across their window geometries (tests/session_geometry.py: one-frame chunks to the 16-bucket window) against
the FP64 / torch-CPU oracle, at the tightness the headline geometry is held to.

  a. FP32, base-16 models, every geometry, ceil(Tw / n_feat) + 4 steps (at least 12) through submit / collect with 3 in flight, on
     tests/gated_speech.py's stream with pauses at a 60 dB gate (partial masks walk the stage-1 buckets) and with no gate (the top
     bucket on every step): stream_compare.compare_stream_pulse_aware -- per-step lengths, the synthesizer's rows (voicing exact, f0 1e-6
     relative, envelope per-frame log-L2 2e-3, ap 1e-6), the session against the oracle synthesizer on the device's rows to 1e-9, and
     against the oracle stream to 1e-6 outside a moved pulse;
  b. FP16, base-64 models, stage 1 fused, at G3 and G7: the same at the FP16 tolerances (envelope 1e-2 / 6e-2, sample RMSE 1e-3,
     log-STFT distance 0.1), without the 1e-9 step (the session's stage-2 plans are banded, its sums ordered unlike the per-op calls');
  c. FP32 groups of two members on different inputs at G2 and G7: each member bitwise its session alone;
  d. noise suppression at G1 (120-sample steps: most finish no 128-sample filter frame), G2 and G7, and device input rates of 48 kHz
     at G1 and 44.1 kHz at G2: bitwise a native session fed concat(zeros(D), filtered or resampled input);
  e. the first window the stage-1 graph table cannot hold (Tw 1920, 17 buckets) is refused at creation, launching nothing and leaving
     device memory where it was.
"""
import math

import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import wave_io

from . import gated_speech as gs
from . import session_geometry as sg
from .stream_compare import DeviceRowsOracle, compare_stream_pulse_aware, run_stream
from .test_gpu_denoise import _filtered_input, _noisy, _profile
from .test_gpu_f0_control import _push
from .test_gpu_parity import _load
from .test_gpu_silence_gate_paths import _run_group, _run_session

pytestmark = pytest.mark.gpu

FS = sg.FS
GEOS = sg.GEOMETRIES
IDS = [g.id for g in GEOS]


def _steps(geo):
    return max(12, math.ceil(geo.Tw / geo.n_feat) + 4)


def _stream(geo, steps, stream=710):
    return gs.stream_with_pauses(seconds=max(10.5, (steps + 1) * geo.buffer_time), stream=stream)


def _chunks(x, geo, steps, n=None):
    n = geo.n_wave if n is None else n
    assert len(x) >= steps * n
    return [np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32) for k in range(steps)]


def _bucket_table(label, geo, x, steps, thr):
    """the oracle's (T_eff, bucket) of every step, printed; the gate's margins hold"""
    rows = gs.step_counts(x, steps, thr, geo.buffer_time, geo.extra[1])
    assert min(m for _, _, m in rows) >= gs.MIN_MARGIN_DB
    print(f'{label}: Tw {geo.Tw} Tp {geo.Tp} ({geo.buckets} buckets); step: T_eff (bucket) '
          + ' '.join(f'{k}:{c}({b})' for k, (c, b, _) in enumerate(rows)) + f'; buckets visited {sorted({b for _, b, _ in rows})}')
    return rows


def _oracle(paths, geo, chunks, thr, stats):
    p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
    return run_stream(opipe.StreamOracle(opipe.PathConfig(threshold_db=thr), p1, p2, stats, buffer_time=geo.buffer_time, extra=geo.extra,
                                         backend='torch'), chunks)


def _device_rows(engine, geo, chunks, thr):
    return run_stream(DeviceRowsOracle(engine, opipe.PathConfig(threshold_db=thr), geo.buffer_time, geo.extra), chunks)


@pytest.fixture
def small(engine, small_models):
    ac, sr, f0c = _load(engine, small_models)
    yield f0c.stats()
    engine.set_precision('fp16')


@pytest.fixture
def full(engine, full_models):
    ac, sr, f0c = _load(engine, full_models)
    engine.set_precision('fp16')
    yield f0c.stats()
    engine.set_stage1_fused(True)
    engine.set_precision('fp16')


# ---- a. FP32, every geometry --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('thr', [60.0, None], ids=['gate60', 'nogate'])
@pytest.mark.parametrize('geo', GEOS, ids=IDS)
def test_fp32_session_is_the_oracle_at_every_geometry(engine, small_models, small, geo, thr):
    steps = _steps(geo)
    x = _stream(geo, steps)
    label = f'{geo.id} fp32 base-16, gate {thr}'
    buckets = [b for _, b, _ in _bucket_table(label, geo, x, steps, thr)]
    assert max(buckets) <= geo.buckets - 1
    if thr is None:
        assert buckets == [geo.buckets - 1] * steps           # every frame effective: the top bucket on every step
    chunks = _chunks(x, geo, steps)
    engine.set_precision('fp32')
    outs, _ = _run_session(engine, geo.session_config(thr), chunks)
    compare_stream_pulse_aware(label, outs, _oracle(small_models, geo, chunks, thr, small), _device_rows(engine, geo, chunks, thr),
                               'small', 'fp32')


# ---- b. FP16, base-64 models --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('geo', [sg.BY_ID['G3'], sg.BY_ID['G7']], ids=['G3', 'G7'])
def test_fp16_full_models_fused(engine, full_models, full, geo):
    steps = _steps(geo)
    x = _stream(geo, steps)
    label = f'{geo.id} fp16 base-64 stage 1 fused, gate 60'
    _bucket_table(label, geo, x, steps, 60.0)
    chunks = _chunks(x, geo, steps)
    assert engine.set_stage1_fused(True) >= 1, 'fused stage-1 kernel unavailable on this device'
    outs, _ = _run_session(engine, geo.session_config(60.0), chunks)
    compare_stream_pulse_aware(label, outs, _oracle(full_models, geo, chunks, 60.0, full), _device_rows(engine, geo, chunks, 60.0),
                               'full', 'fp16', lsd_tol=0.1)


# ---- c. groups ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('geo', [sg.BY_ID['G2'], sg.BY_ID['G7']], ids=['G2', 'G7'])
def test_group_members_are_their_sessions_alone(engine, small_models, small, geo):
    steps = _steps(geo)
    members = [_chunks(_stream(geo, steps, stream=720 + i)[round(off * FS):], geo, steps) for i, off in enumerate((0.0, 0.8))]
    engine.set_precision('fp32')
    grouped = _run_group(engine, geo.session_config(60.0), members)
    for i, m in enumerate(members):
        alone, _ = _run_session(engine, geo.session_config(60.0), m)
        assert sum(len(o) for o in alone) > 0 and float(np.abs(np.concatenate(alone)).max()) > 1e-2
        assert [len(o) for o in grouped[i]] == [len(o) for o in alone], i
        assert all(np.array_equal(a, b) for a, b in zip(grouped[i], alone)), i
        print(f'{geo.id} group member {i}: {steps} steps, {sum(len(o) for o in alone)} samples, bitwise its session alone')


# ---- d. noise suppression and device input rates ------------------------------------------------------------------------------
def _session(engine, geo, created):
    sid = engine.session_create(geo.session_config(60.0))
    created.append(sid)
    return sid


@pytest.fixture
def created(engine):
    sids = []
    yield sids
    for sid in sids:
        engine.session_destroy(sid)


@pytest.mark.parametrize('geo,steps,lead', [(sg.BY_ID['G1'], 80, 0.05), (sg.BY_ID['G2'], 24, 0.3), (sg.BY_ID['G7'], 6, 0.5)],
                         ids=['G1', 'G2', 'G7'])
def test_denoised_session_is_the_filtered_stream_bitwise(engine, small_models, small, created, geo, steps, lead):
    engine.set_precision('fp32')
    x = _noisy((steps + 1) * geo.buffer_time, stream=731, lead=lead)
    phi = _profile(x, count=min(80, round(lead * FS) // 128 - 3))
    a = _session(engine, geo, created)
    engine.session_denoise(a)
    engine.session_set_noise_profile(a, phi)
    geo_a = engine.session_io_geometry(a)
    assert geo_a['n_in'] == geo.n_wave and geo_a['delay_in'] == 511
    ref_in = _filtered_input(engine, x[:steps * geo.n_wave], 20.0, phi)
    out_a = _push(engine, a, _chunks(x, geo, steps))
    out_b = _push(engine, _session(engine, geo, created), _chunks(ref_in, geo, steps))
    plain = _push(engine, _session(engine, geo, created), _chunks(x, geo, steps))
    n = sum(len(o) for o in out_a)
    print(f'{geo.id} noise suppression: {steps} steps of {geo.n_wave} samples, {n} samples out, bitwise the native session on the '
          f'filtered input')
    assert n > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert [len(o) for o in out_a] == [len(o) for o in out_b] and all(np.array_equal(p, q) for p, q in zip(out_a, out_b))
    assert not all(np.array_equal(p, q) for p, q in zip(out_a, plain))         # the filter does something


@pytest.mark.parametrize('geo,rate,n_in', [(sg.BY_ID['G1'], 48000, 240), (sg.BY_ID['G2'], 44100, 2205)], ids=['G1-48k', 'G2-44k1'])
def test_device_input_rate_is_the_resampled_stream_bitwise(engine, small_models, small, created, geo, rate, n_in):
    engine.set_precision('fp32')
    steps = 60 if geo.id == 'G1' else 24
    x24 = gs.stream_with_pauses(seconds=(steps + 2) * geo.buffer_time + 0.2, stream=741)
    x = wave_io.resample(x24, FS, rate, engine)
    n, _, D = wave_io.stream_input_geometry(rate, FS, geo.buffer_time)
    assert n == n_in
    a = _session(engine, geo, created)
    engine.session_set_input_rate(a, rate)
    g = engine.session_io_geometry(a)
    assert (g['n_in'], g['delay_in'], g['in_rate']) == (n_in, D, rate)
    g_ = math.gcd(rate, FS)
    up, down = FS // g_, rate // g_
    model = np.concatenate([np.zeros(D, np.float32), engine.resample_poly(x, up, down, wave_io.resample_filter(up, down))]).astype(np.float32)
    out_a = _push(engine, a, _chunks(x, geo, steps, n_in))
    out_b = _push(engine, _session(engine, geo, created), _chunks(model, geo, steps))
    m = sum(len(o) for o in out_a)
    print(f'{geo.id} input at {rate} Hz: {steps} steps of {n_in} samples (delay {D}), {m} samples out, bitwise the native session')
    assert m > 0 and float(np.abs(np.concatenate(out_a)).max()) > 1e-2
    assert [len(o) for o in out_a] == [len(o) for o in out_b] and all(np.array_equal(p, q) for p, q in zip(out_a, out_b))


# ---- e. the bucket limit ------------------------------------------------------------------------------------------------------
def test_a_window_beyond_the_bucket_table_is_refused_at_creation(engine, small_models, small):
    import torch
    too_long = sg.TOO_LONG
    assert (too_long.Tw, too_long.Tp, too_long.buckets) == (1920, 2048, 17)
    engine.synchronize()
    free, before = torch.cuda.mem_get_info()[0], engine.launch_count
    with pytest.raises(Exception, match='window too long for the stage-1 graph table'):
        engine.session_create(too_long.session_config())
    engine.synchronize()
    assert engine.launch_count == before
    assert abs(torch.cuda.mem_get_info()[0] - free) < 2**20, (free, torch.cuda.mem_get_info()[0])
    # the largest window the table holds is accepted (and steps: part a)
    sid = engine.session_create(sg.BY_ID['G9'].session_config())
    engine.session_destroy(sid)
