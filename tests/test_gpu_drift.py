"""The clock drift stage on the device (ryk_drift_*, DESIGN.md §4l) against the FP64 oracle (tests/drift_oracle.py).

  * ryk_drift_resample is the oracle bit for bit at 24, 44.1 and 48 kHz for ppm in {-1000, -37.5, 0, 12.3, 500, 1000};
  * ryk_drift_push at seeded random sizes, with setting changes between pushes, is the oracle's stream; the totals are the oracle's;
  * RealtimePipeline through run.audio_loop at the headline configuration with drift=250 plays the oracle's drift of what the same
    pipeline plays without it, and with echo_cancel the far end is the one without drift;
  * a snapshot taken mid-stream continues bit for bit on another engine; a pipeline blob with DRFT round-trips;
  * one kernel per push; refusals change nothing; create / destroy cycles return memory.
"""
import functools

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io
from realtime_yukarin_b200.engine import Engine, RykError, describe_snapshot

from . import drift_oracle as D
from .test_gpu_f0_control import EXTRA, FS, T
from .test_gpu_launch_count import _kernel_events, _run_child

pytestmark = pytest.mark.gpu

PPMS = (-1000.0, -37.5, 0.0, 12.3, 500.0, 1000.0)
_second = {}


def _signal(rate, seconds, stream):
    x = synthetic.synthetic_speech(seconds, stream=stream)
    if rate != FS:
        x = np.interp(np.arange(round(len(x) * rate / FS)) * FS / rate, np.arange(len(x)), x)
    return np.asarray(x, np.float64)


def _other_engine():
    if 'e' not in _second:
        _second['e'] = Engine(device=0)
    return _second['e']


# ---- 1 --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('rate', [24000, 44100, 48000])
def test_resample_is_the_oracle_bit_for_bit(engine, rate):
    x = _signal(rate, 1.0, stream=rate // 100)
    for ppm in PPMS:
        got = engine.drift_resample(x, ppm)
        want = D.resample(x, ppm)
        assert len(got) == len(want) and np.array_equal(got, want), ppm
    assert np.array_equal(engine.drift_resample(x, 0.0), np.concatenate([np.zeros(D.W), x]))


# ---- 2 --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seed', [11, 12])
def test_streamed_pushes_are_the_oracle_stream(engine, seed):
    rng = np.random.default_rng(seed)
    x = _signal(48000, 3.0, stream=seed)
    did = engine.drift_create(20000, 1000.0)
    ref = D.DriftStream(0.0)
    try:
        a = 0
        while a < len(x):
            if rng.random() < 0.5:
                ppm = float(rng.choice([rng.uniform(-1000, 1000), *PPMS]))
                engine.drift_set(did, ppm)
                ref.set(ppm)
                assert engine.drift_get(did) == (ppm, D.inc_of(ppm))
            n = int(rng.choice([0, 1, 31, 32, 33, int(rng.integers(0, 20001))]))
            got, want = engine.drift_push(did, x[a:a + n]), ref.push(x[a:a + n])
            assert np.array_equal(got, want), a
            a += n
            assert engine.drift_stats(did) == (ref.consumed, ref.produced)
    finally:
        engine.drift_destroy(did)


# ---- 3 --------------------------------------------------------------------------------------------------------------------------
def test_the_pipeline_plays_the_oracle_drift_of_its_plain_output(engine, full_models, monkeypatch):
    from realtime_yukarin_b200 import run as run_mod
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import RealtimePipeline
    from .test_gpu_parity import _load
    _load(engine, full_models)
    engine.set_precision('fp16')
    config = Config(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                    extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                    output_silent_threshold=80.0, encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2],
                    **{k: full_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                   'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})
    n, steps = config.in_audio_chunk, 16
    x = synthetic.synthetic_speech((steps + 1) * T, stream=613).astype(np.float32)
    fars = []
    real_ref = engine.session_echo_reference
    monkeypatch.setattr(engine, 'session_echo_reference', lambda sid, far: fars[-1].append(np.array(far)) or real_ref(sid, far))

    def play(**kw):
        fars.append([])
        pipe = RealtimePipeline(config, engine=engine, **kw)
        # every chunk is finished before process() returns: otherwise a chunk the device has not finished in time plays as zeros and
        # a later one takes its place, so what is played, and the far end made from it, would move with the device's timing
        pipe.process = functools.partial(pipe.process, block=True)
        played, pos = [], [0]

        def read_chunk():
            k = pos[0]
            if k >= steps:
                return None
            pos[0] = k + 1
            return x[k * n:(k + 1) * n]
        try:
            assert run_mod.audio_loop(pipe, read_chunk, played.append) == steps
            played += pipe.drain()
        finally:
            pipe.close()
        return np.concatenate(played)
    for echo in (False, True):
        kw = dict(echo_cancel=True, echo_taps=8) if echo else {}
        plain = play(**kw)
        drifted = play(drift=250.0, **kw)
        assert np.any(plain != 0)
        want = D.resample(plain.astype(np.float64), 250.0).astype(np.float32)
        assert drifted.dtype == np.float32 and np.array_equal(drifted, want), echo
        if echo:
            assert len(fars[-1]) == len(fars[-2]) == steps and all(np.array_equal(a, b) for a, b in zip(fars[-2], fars[-1]))


# ---- 4 --------------------------------------------------------------------------------------------------------------------------
def test_a_snapshot_continues_on_another_engine(engine):
    x = _signal(48000, 2.0, stream=77)
    src = engine.drift_create(14400, 500.0)
    try:
        engine.drift_set(src, -321.5)
        for k in range(5):
            engine.drift_push(src, x[k * 14400:(k + 1) * 14400])
        engine.drift_set(src, 123.25)                                   # a setting made after the last push travels too
        blob = engine.drift_snapshot(src)
        d = describe_snapshot(blob)
        assert d['kind'] == 'drift' and [t for t, _ in d['sections']] == ['DCNF', 'DSTA', 'DHIS']
        assert d['config']['max_in'] == 14400 and d['config']['max_ppm'] == 500.0 and d['config']['pushed'] == 5
        for dst_engine in (engine, _other_engine()):
            dst = dst_engine.drift_restore(blob)
            try:
                assert dst_engine.drift_get(dst) == engine.drift_get(src)
                assert dst_engine.drift_stats(dst) == engine.drift_stats(src)
                chunks = [x[a:a + 9000] for a in range(72000, len(x), 9000)]
                ref = engine.drift_restore(blob)                        # a second copy on the source engine: the reference
                try:
                    for c in chunks:
                        assert np.array_equal(engine.drift_push(ref, c), dst_engine.drift_push(dst, c))
                finally:
                    engine.drift_destroy(ref)
            finally:
                dst_engine.drift_destroy(dst)
        # the oracle continues the same way
        o = D.DriftStream(-321.5)
        for k in range(5):
            o.push(x[k * 14400:(k + 1) * 14400])
        o.set(123.25)
        dst = _other_engine().drift_restore(blob)
        try:
            assert np.array_equal(_other_engine().drift_push(dst, x[72000:86400]), o.push(x[72000:86400]))
        finally:
            _other_engine().drift_destroy(dst)
    finally:
        engine.drift_destroy(src)


def test_a_pipeline_blob_with_drift_round_trips(engine, full_models):
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import RealtimePipeline, unpack_pipeline
    from .test_gpu_parity import _load
    _load(engine, full_models)
    engine.set_precision('fp16')
    config = Config(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                    extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.5, input_silent_threshold=60.0,
                    output_silent_threshold=80.0, encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2],
                    **{k: full_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                   'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})
    n = config.in_audio_chunk
    x = synthetic.synthetic_speech(13 * T, stream=615).astype(np.float32)
    chunks = [x[k * n:(k + 1) * n] for k in range(12)]
    src = RealtimePipeline(config, engine=engine, drift='auto', drift_max_ppm=300.0)
    try:
        for k, c in enumerate(chunks[:6]):
            src.process(c)
            for j in range(6):                                          # past the controller's warm-up and set-point
                src.update_drift(20000 + 300 * k + 50 * j)
        assert src.drift_stats()['ppm'] != 0.0
        src.drain()
        blob = src.snapshot()
        assert [t for t, _ in describe_snapshot(blob)['sections']] == ['SESS', 'RBLK', 'PIPE', 'DRFT']
        parts = unpack_pipeline(blob)
        assert describe_snapshot(parts['drift'])['kind'] == 'drift'
        assert parts['host']['drift']['controller'] == src._drift_ctl.state()
        dst = RealtimePipeline.restore(blob, config, engine=_other_engine_with_models(full_models))
        try:
            assert dst.drift_auto and dst.drift_stats() == src.drift_stats()
            for k, c in enumerate(chunks[6:]):
                a, b = src.process(c, block=True), dst.process(c, block=True)
                assert np.array_equal(a, b), k
                assert src.update_drift(22000 - 250 * k) == dst.update_drift(22000 - 250 * k)
            assert all(np.array_equal(a, b) for a, b in zip(src.drain(), dst.drain()))
            ps, pd = unpack_pipeline(src.snapshot()), unpack_pipeline(dst.snapshot())
            assert ps['drift'] == pd['drift'] and ps['host'] == pd['host']
        finally:
            dst.close()
    finally:
        src.close()


def _other_engine_with_models(full_models):
    from .test_gpu_parity import _load
    e = _other_engine()
    if not _second.get('models'):
        _load(e, full_models)
        _second['models'] = True
    e.set_precision('fp16')
    return e


# ---- 5 --------------------------------------------------------------------------------------------------------------------------
def _launch_window(out_dir):
    """Child process of the launch test: returns the names of the kernels the profiler saw over 12 pushes."""
    from torch.profiler import ProfilerActivity, profile
    from realtime_yukarin_b200.engine import default_engine
    engine = default_engine()
    did = engine.drift_create(14400, 500.0)
    engine.drift_set(did, 250.0)
    x = _signal(48000, 4.0, stream=5)
    engine.drift_push(did, x[:14400])                                  # first launch outside the window
    engine.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(1, 13):
            engine.drift_push(did, x[k * 14400:(k + 1) * 14400])
        engine.synchronize()
    return [e['name'] for e in _kernel_events(prof, out_dir / 'trace.json')]


def test_one_kernel_per_push(tmp_path):
    names = _run_child(tmp_path, 'test_gpu_drift', '_launch_window')
    print(f'kernels over 12 pushes: {len(names)}')
    assert len(names) == 12 and all('k_drift' in s for s in names)


def test_refusals_change_nothing(engine):
    import ctypes
    x = _signal(24000, 0.5, stream=9)
    did = engine.drift_create(7200, 200.0)
    try:
        engine.drift_set(did, 150.0)
        engine.drift_push(did, x[:7200])
        before = (engine.drift_get(did), engine.drift_stats(did), engine.drift_snapshot(did))
        for ppm in (200.5, -201.0, float('nan'), float('inf')):
            with pytest.raises(RykError):
                engine.drift_set(did, ppm)
        lib = engine.lib
        y = np.empty(7200, np.float64)
        n = ctypes.c_int()
        xs = np.ascontiguousarray(x[:7200])
        for cap, count in ((7200 + 2 + 1, 7200), (7200, 7200), (10, 7201)):     # too small, and more samples than max_in
            rc = lib.ryk_drift_push(engine._h, did, xs.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), count,
                                    y.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), cap, ctypes.byref(n))
            assert rc < 0
        with pytest.raises(RykError):
            engine.drift_create(7200, 200.0, table=np.zeros(100))
        T = wave_io.drift_filter()
        for bad_shape in ((256, 16), (512, 8)):
            assert lib.ryk_drift_create(engine._h, 100, ctypes.c_double(100.0), T.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                        bad_shape[0], bad_shape[1], ctypes.byref(n)) < 0
        for max_ppm in (0.0, -1.0, 2000.5):
            with pytest.raises(RykError):
                engine.drift_create(7200, max_ppm)
        bad_table = T.copy()
        bad_table[5] = np.nan
        with pytest.raises(RykError):
            engine.drift_create(7200, 200.0, table=bad_table)
        blob = before[2]
        corrupt = bytearray(blob)
        corrupt[-3] ^= 1
        rid = engine.reblock_create(2400, 4800, 80.0)
        for bad in (bytes(corrupt), blob[:-8], b'', engine.reblock_snapshot(rid)):
            with pytest.raises(RykError):
                engine.drift_restore(bad)
        engine.reblock_destroy(rid)
        assert (engine.drift_get(did), engine.drift_stats(did), engine.drift_snapshot(did)) == before
        probe = engine.drift_create(100, 10.0)                          # the refused calls made no drift object
        assert probe == did + 1
        engine.drift_destroy(probe)
    finally:
        engine.drift_destroy(did)


def test_cycles_return_memory(engine):
    import torch
    free = {}
    x = _signal(48000, 1.0, stream=3)
    for cycle in range(13):
        did = engine.drift_create(48000, 1000.0)
        engine.drift_set(did, 999.0)
        engine.drift_push(did, x)
        engine.drift_restore(engine.drift_snapshot(did))
        engine.drift_destroy(did)
        engine.drift_destroy(did + 1)
        if cycle in (2, 12):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[12]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 10 drift create / restore / destroy cycles')
    assert abs(grown) < 2.0
