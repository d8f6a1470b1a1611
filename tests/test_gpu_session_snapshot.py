"""Moving a streaming session (ryk_session_snapshot / _restore, the re-blocker pair, RealtimePipeline.snapshot / restore) at the headline
configuration: 0.3 s chunks, extras (0, 0.5, 0), base-64 synthetic models.

The core assertion: session A runs k steps, its snapshot is restored as B, then A and B are fed the same next chunks (and the same far
end) and return the same samples bit for bit.
  * k covers both parities, every k % 6, the first two steps (before every graph copy is captured) and one run past a synthesizer
    noise-ring top-up and an event-ring wrap;
  * with every optional stage on together and with each alone, settings changed just before the snapshot included;
  * on the same engine, on a second engine of the same device, and on a second device when one is visible;
  * group members restored into an identically built group; the pipeline with its re-blocker;
  * refusals leave both engines unchanged; a snapshot changes nothing for the source; cycles return device memory.
"""

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import Engine, RykError

from .test_gpu_f0_control import FS, N, T, _cfg, _new_voice, _same, made, second_voice_files  # noqa: F401
from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

_engines = {}


def _engine_on(device, full_models):
    """A second engine (kept for the process: an engine's destruction also frees the process's CREPE model) with the models loaded."""
    if device not in _engines:
        e = Engine(device=device)
        _load(e, full_models)
        _engines[device] = e
    e = _engines[device]
    e.set_precision('fp16')
    return e


def _speech(steps, stream, n=N, rate=FS):
    x = synthetic.synthetic_speech((steps + 1) * T, stream=stream)
    if rate != FS:
        x = np.interp(np.arange(round(len(x) * rate / FS)) * FS / rate, np.arange(len(x)), x)
    return [np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32) for k in range(steps)]


class Stream:
    """One stream's inputs: mic chunks and, with echo cancellation, far-end chunks; `step(e, sid, k)` pushes chunk k."""

    def __init__(self, steps, stream, rate=FS, echo=False):
        n = round(T * rate)
        self.mic = _speech(steps, stream, n, rate)
        self.far = _speech(steps, stream + 1000, n, rate) if echo else None

    def step(self, e, sid, k, buf):
        if self.far is not None:
            e.session_echo_reference(sid, self.far[k] * np.float32(0.5))
        return e.session_push(sid, self.mic[k], buf).copy()


STAGES = ('denoise', 'denoise_learning', 'echo', 'agc', 'limiter', 'f0', 'formant', 'rates48')


def _setup(e, sid, stages):
    """enable `stages` on a fresh session"""
    if 'rates48' in stages:
        e.session_set_input_rate(sid, 48000)
        e.session_set_output_rate(sid, 48000)
    if 'denoise' in stages or 'denoise_learning' in stages:
        e.session_denoise(sid)
        e.session_set_denoise(sid, 18.0)
        e.session_denoise_learn(sid, frames=40 if 'denoise' in stages else 5000)    # learned after the first steps / still learning
    if 'echo' in stages:
        e.session_echo_cancel(sid, taps=16, delay_ms=0.0)
    if 'agc' in stages:
        e.session_agc(sid, -20.0, 20.0, -60.0)
    if 'limiter' in stages:
        e.session_limiter(sid, lookahead_ms=5.0, hold_ms=20.0)
        e.session_set_limiter(sid, -20.0, gain=1.0)
    if 'f0' in stages:
        e.session_f0_measure(sid)
        e.session_f0_follow(sid, True, min_voiced_frames=50)
    if 'formant' in stages:
        e.session_set_formant(sid, ratio=1.15)


def _late_settings(e, sid, stages):
    """settings changed just before a snapshot: they must land on the restored session's next step"""
    e.session_set_f0_map(sid, semitones=2.0)
    if 'denoise' in stages or 'denoise_learning' in stages:
        e.session_set_denoise(sid, 9.0)
    if 'echo' in stages:
        e.session_set_echo_suppression(sid, 6.0)
    if 'agc' in stages:
        e.session_set_agc(sid, target_db=-24.0)
    if 'limiter' in stages:
        e.session_set_limiter(sid, -12.0, gain=1.5)
    if 'formant' in stages:
        e.session_set_formant(sid, ratio=0.9)


def _move_and_compare(e, made, k, stages=(), voice=0, dst=None, after=3, late=True, f0_method=None, stream=700):
    """A runs k steps; B = restore(snapshot(A)) on dst; A and B then get the same `after` chunks: bitwise the same outputs"""
    dst = dst or e
    rate = 48000 if 'rates48' in stages else FS
    x = Stream(k + after, stream + k, rate, echo='echo' in stages)
    a = made.create(voice=voice, f0_method=f0_method)
    _setup(e, a, stages)
    buf = np.empty(e.session_io_geometry(a)['max_out'])
    for j in range(k):
        x.step(e, a, j, buf)
    if late:
        _late_settings(e, a, stages)
    blob = e.session_snapshot(a)
    b = dst.session_restore(blob, voice=voice)
    if dst is e:
        made.sids.append(b)
    try:
        assert dst.session_io_geometry(b) == e.session_io_geometry(a)
        outs_a = [x.step(e, a, j, buf) for j in range(k, k + after)]
        outs_b = [x.step(dst, b, j, buf) for j in range(k, k + after)]
        assert _same(outs_a, outs_b), (k, stages, [int(np.count_nonzero(p != q)) if len(p) == len(q) else (len(p), len(q))
                                                    for p, q in zip(outs_a, outs_b)])
        assert sum(len(o) for o in outs_a) > 0
        if 'f0' in stages:
            assert e.session_f0_measured(a) == dst.session_f0_measured(b)
    finally:
        if dst is not e:
            dst.session_destroy(b)
    return blob


# ---- 1: step counts ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', range(8))
def test_restored_session_continues_bitwise(engine, made, k):
    _move_and_compare(engine, made, k)


@pytest.mark.parametrize('k', range(8))
def test_every_stage_on_continues_bitwise(engine, made, k):
    _move_and_compare(engine, made, k, stages=STAGES[:1] + STAGES[2:])


def test_past_a_noise_ring_top_up_and_an_event_ring_wrap(engine, made):
    # the synthesizer tops its noise ring up every 2^21 samples (step 291 at 0.3 s chunks); the restored session's first steps run it
    _move_and_compare(engine, made, 290, after=4, late=False)


# ---- 2: each stage alone -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('stage', STAGES)
@pytest.mark.parametrize('k', [1, 4])
def test_each_stage_alone_continues_bitwise(engine, made, stage, k):
    _move_and_compare(engine, made, k, stages=(stage,))


def test_a_voice_other_than_zero(engine, made, full_models):
    v = _new_voice(engine, made, full_models)
    _move_and_compare(engine, made, 3, voice=v)


def test_crepe_with_seeded_weights(engine, made, tmp_path):
    from realtime_yukarin_b200 import crepe as pcrepe
    pcrepe.load_crepe_model(synthetic.write_crepe_model(tmp_path, seed=5, capacity='tiny'), engine)
    pcrepe.set_session_rate(FS, engine)
    _move_and_compare(engine, made, 3, f0_method='crepe')
    _move_and_compare(engine, made, 4, stages=('denoise', 'agc'), f0_method='crepe')


# ---- 3: destinations ------------------------------------------------------------------------------------------------------------
def test_to_a_second_engine_on_the_same_device(engine, made, full_models):
    dst = _engine_on(0, full_models)
    for k in (2, 5):
        _move_and_compare(engine, made, k, stages=STAGES[:1] + STAGES[2:], dst=dst)
    _move_and_compare(engine, made, 3, dst=dst)


def test_to_a_second_device(engine, made, full_models):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip('one CUDA device visible: a move to another device needs two')
    dst = _engine_on(1, full_models)
    _move_and_compare(engine, made, 3, stages=STAGES[:1] + STAGES[2:], dst=dst)


def test_group_members_restored_into_an_identical_group(engine, made, full_models):
    dst = _engine_on(0, full_models)
    k, after = 5, 3
    xs = [Stream(k + after, 760 + i) for i in range(2)]
    src = [made.create() for _ in range(2)]
    engine.session_agc(src[1], -20.0, 20.0, -60.0)
    g = engine.group_create(src)
    made.gids.append(g)
    outs = [np.empty(engine.session_io_geometry(src[0])['max_out']) for _ in src]
    for j in range(k):
        engine.group_collect(g, engine.group_submit(g, [x.mic[j] for x in xs]), outs)
    blobs = [engine.session_snapshot(s) for s in src]
    dsts = [dst.session_restore(b) for b in blobs]
    gd = dst.group_create(dsts)
    try:
        for j in range(k, k + after):
            a = [o.copy() for o in engine.group_collect(g, engine.group_submit(g, [x.mic[j] for x in xs]), outs)]
            b = [o.copy() for o in dst.group_collect(gd, dst.group_submit(gd, [x.mic[j] for x in xs]), outs)]
            assert _same(a, b), j
    finally:
        dst.group_destroy(gd)
        for s in dsts:
            dst.session_destroy(s)


# ---- 4: the pipeline -----------------------------------------------------------------------------------------------------------
def test_pipeline_snapshot_and_restore(engine, made, full_models):
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import RealtimePipeline
    config = Config(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=T,
                    extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=0.8, output_scale=1.5, input_silent_threshold=60.0,
                    output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0,
                    **{k: full_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                   'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})
    x = _speech(12, 780)
    for dst_engine in (engine, _engine_on(0, full_models)):
        src = RealtimePipeline(config, engine=engine, denoise=12.0, learn_noise=0.2, echo_cancel=True, echo_taps=8, limiter=-6.0,
                               agc=-22.0)
        try:
            for c in x[:5]:
                src.process(c)
            src.drain()
            blob = src.snapshot()
            dst = RealtimePipeline.restore(blob, config, engine=dst_engine)
            try:
                for c in x[5:]:
                    a, b = src.process(c, block=True), dst.process(c, block=True)
                    assert np.array_equal(a, b)
                assert _same(src.drain(), dst.drain())
            finally:
                dst.close()
        finally:
            src.close()


# ---- 5: refusals, the source, memory ---------------------------------------------------------------------------------------------
def test_refusals_change_nothing(engine, made, full_models):
    import torch
    x = Stream(6, 790)
    a, twin = made.create(), made.create()
    buf = np.empty(engine.session_io_geometry(a)['max_out'])
    for j in range(2):
        x.step(engine, a, j, buf)
        x.step(engine, twin, j, buf)
    t = engine.session_submit(a, x.mic[2])
    with pytest.raises(RykError, match='in flight'):
        engine.session_snapshot(a)
    engine.session_collect(a, t, buf)
    x.step(engine, twin, 2, buf)
    blob = engine.session_snapshot(a)
    dst = _engine_on(0, full_models)
    small = _new_voice(engine, made, second_voice_files_small(full_models))
    engine.synchronize()
    dst.synchronize()
    free = torch.cuda.mem_get_info()[0]
    bad = bytearray(blob)
    bad[len(bad) // 2] ^= 1
    cases = [(dst, bytes(bad), 0, 'checksum'), (dst, blob[:-16], 0, 'truncated'), (engine, blob, small, 'channels')]
    dst.set_precision('fp32')
    try:
        with pytest.raises(RykError, match='precision'):
            dst.session_restore(blob)
    finally:
        dst.set_precision('fp16')
    for e, b, voice, needle in cases:
        with pytest.raises(RykError, match=needle):
            e.session_restore(b, voice=voice)
    engine.synchronize()
    dst.synchronize()
    assert torch.cuda.mem_get_info()[0] == free
    # the source runs on as its twin that was never snapshotted
    assert _same([x.step(engine, a, j, buf) for j in range(3, 6)], [x.step(engine, twin, j, buf) for j in range(3, 6)])


def second_voice_files_small(full_models):
    """a voice whose stage-2 net is narrower (base 16) than the snapshot's: a shape mismatch"""
    import tempfile
    return synthetic.write_synthetic_models(tempfile.mkdtemp(prefix='ryk_snap_small_'), seed=9, base1=64, base2=16)


def test_a_snapshot_changes_nothing_for_the_source(engine, made):
    stages = STAGES[:1] + STAGES[2:]
    x = Stream(9, 800, rate=48000, echo=True)
    a, twin = made.create(), made.create()
    for s in (a, twin):
        _setup(engine, s, stages)
    buf = np.empty(engine.session_io_geometry(a)['max_out'])
    out_a, out_t = [], []
    for j in range(9):
        if j % 2 == 0:
            engine.session_snapshot(a)
        out_a.append(x.step(engine, a, j, buf))
        out_t.append(x.step(engine, twin, j, buf))
    assert _same(out_a, out_t)


def test_cycles_return_device_memory(engine, made, full_models):
    import torch
    dst = _engine_on(0, full_models)
    x = Stream(3, 810)
    free = {}
    for cycle in range(1, 6):
        a = engine.session_create(_cfg())
        _setup(engine, a, ('denoise', 'agc', 'limiter'))
        buf = np.empty(engine.session_io_geometry(a)['max_out'])
        for j in range(3):
            x.step(engine, a, j, buf)
        b = dst.session_restore(engine.session_snapshot(a))
        rid = dst.reblock_create(N, 2 * N, 80.0)
        r2 = dst.reblock_restore(dst.reblock_snapshot(rid))
        dst.session_destroy(b)
        dst.reblock_destroy(rid)
        dst.reblock_destroy(r2)
        engine.session_destroy(a)
        if cycle in (2, 5):
            engine.synchronize()
            dst.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    assert free[5] == free[2], free


def test_reblock_snapshot_continues_bitwise(engine):
    rng = np.random.default_rng(3)
    chunk = 2400
    a = engine.reblock_create(chunk, 4096, 80.0)
    try:
        pieces = [rng.normal(0, 0.1, rng.integers(0, 4096)) for _ in range(12)]
        for p in pieces[:5]:
            engine.reblock_push(a, p)
        b = engine.reblock_restore(engine.reblock_snapshot(a))
        try:
            for p in pieces[5:]:
                ra, rb = engine.reblock_push(a, p), engine.reblock_push(b, p)
                assert ra[0] == rb[0] and ra[2] == rb[2] and (ra[1] is None) == (rb[1] is None)
                if ra[1] is not None:
                    assert np.array_equal(ra[1], rb[1])
        finally:
            engine.reblock_destroy(b)
    finally:
        engine.reblock_destroy(a)
