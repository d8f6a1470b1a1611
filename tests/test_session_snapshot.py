"""Moving a session without a GPU: the snapshot container as ryk_snapshot_describe reads it (header, FNV-1a-64 checksum, section
walk, refusals), the recorded configuration of a session blob, the pipeline blob that packs the session's and the re-blocker's blobs
with the pipeline's host state, and run.py's --save_state / --load_state options."""
import collections
import ctypes
import struct
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import engine as eng
from realtime_yukarin_b200 import snapshot
from realtime_yukarin_b200.engine import RykError, SessionConfig, SnapshotReblock, SnapshotSession, describe_snapshot


def fnv1a64(data: bytes) -> int:
    h = 0xcbf29ce484222325
    for b in data:
        h = ((h ^ b) * 0x100000001b3) & 0xffffffffffffffff
    return h


def _session_conf(**kw) -> SnapshotSession:
    c = SnapshotSession()
    c.cfg = SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                          buffer_time=0.1, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0, threshold_db=60.0,
                          vocoder_buffer_size=1024)
    c.precision, c.stage1_fused, c.f0_method, c.step = 1, 1, 0, 17
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _session_blob(**kw) -> bytes:
    return snapshot.pack('session', [('CONF', bytes(_session_conf(**kw))), ('HOST', b'\x01' * 24), ('WAVE', b'\x02' * 13)])


def _reblock_blob(chunk=2400, max_in=5120, threshold=80.0) -> bytes:
    c = SnapshotReblock(out_audio_chunk=chunk, max_in=max_in, n_fft=2048, hop=512, threshold_db=threshold, pushed=9)
    return snapshot.pack('reblock', [('RCNF', bytes(c)), ('RSTA', b'\x00' * 12)])


def _reseal(blob: bytearray) -> bytes:
    eng.seal_snapshot(blob)
    return bytes(blob)


def test_container_round_trip_and_layout():
    payloads = [('ABCD', b''), ('EFGH', b'x'), ('IJKL', bytes(range(200))), ('ABCD', b'12345678')]
    blob = snapshot.pack('pipeline', payloads)
    magic, version, kind, total, checksum = struct.unpack_from('<QIIQQ', blob)
    assert blob[:8] == b'RYKSNAP\x00' and version == 1 and kind == 3 and total == len(blob)
    assert checksum == fnv1a64(blob[32:])                       # the header's checksum is FNV-1a-64 of everything after it
    assert len(blob) == 32 + sum(16 + (len(p) + 7) // 8 * 8 for _, p in payloads)
    d = describe_snapshot(blob)
    assert d['kind'] == 'pipeline' and d['version'] == 1 and d['config'] is None
    assert d['sections'] == [(t, len(p)) for t, p in payloads]
    kind, sec = snapshot.unpack(blob)
    assert kind == 'pipeline' and sec == {'ABCD': b'', 'EFGH': b'x', 'IJKL': bytes(range(200))}


def test_describe_reads_the_recorded_configuration():
    d = describe_snapshot(_session_blob(in_rate=48000, in_up=1, in_down=2, echo=1, echo_taps=32, limiter=1, limiter_hold_ms=50.0))
    c = d['config']
    assert d['kind'] == 'session' and c['step'] == 17 and c['cfg']['fs'] == 24000 and c['cfg']['convert_extra_time'] == 0.5
    assert (c['in_rate'], c['in_up'], c['in_down'], c['echo'], c['echo_taps'], c['limiter'], c['limiter_hold_ms']) == (48000, 1, 2, 1, 32, 1, 50.0)
    assert [t for t, _ in d['sections']] == ['CONF', 'HOST', 'WAVE']
    r = describe_snapshot(_reblock_blob())['config']
    assert (r['out_audio_chunk'], r['max_in'], r['n_fft'], r['hop'], r['threshold_db'], r['pushed']) == (2400, 5120, 2048, 512, 80.0, 9)


def test_describe_refuses_corrupt_truncated_and_unknown_blobs():
    blob = _session_blob()
    flipped = bytearray(blob)
    flipped[-3] ^= 0x10
    with pytest.raises(RykError, match='checksum'):
        describe_snapshot(bytes(flipped))
    for cut in (len(blob) - 8, len(blob) - 1, 40, 31, 0):
        with pytest.raises(RykError, match='truncated'):
            describe_snapshot(blob[:cut])
    with pytest.raises(RykError, match='longer'):
        describe_snapshot(blob + b'\x00' * 8)
    other = bytearray(blob)
    struct.pack_into('<I', other, 8, 2)                          # format version 2, sealed again: the checksum is right
    with pytest.raises(RykError, match='unknown format version'):
        describe_snapshot(_reseal(other))
    bad = bytearray(blob)
    bad[0:8] = b'NOTASNAP'
    with pytest.raises(RykError, match='magic'):
        describe_snapshot(bytes(bad))
    walk = bytearray(blob)
    struct.pack_into('<Q', walk, 32 + 8, len(blob))               # the first section claims more bytes than the blob holds
    with pytest.raises(RykError, match='malformed'):
        describe_snapshot(_reseal(walk))
    empty = bytearray(snapshot.pack('session', [('CONF', b'')]))
    with pytest.raises(RykError, match='configuration'):
        describe_snapshot(bytes(empty))


def test_tags_must_be_four_characters():
    with pytest.raises(ValueError):
        snapshot.pack('pipeline', [('ABC', b'')])


# ---- the pipeline blob ---------------------------------------------------------------------------------------------------------
def _config(**kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=24000, output_rate=24000, frame_period=5.0, buffer_time=0.1,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: Path(k) for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                    'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


class MoveEngine:
    """Records what RealtimePipeline.snapshot / restore ask of an engine and hands out the blobs it was given."""

    def __init__(self, session_blob=None, reblock_blob=None):
        self.session_blob, self.reblock_blob = session_blob, reblock_blob
        self.calls = []

    def session_snapshot(self, sid):
        self.calls.append(('session_snapshot', sid))
        return self.session_blob

    def reblock_snapshot(self, rid):
        self.calls.append(('reblock_snapshot', rid))
        return self.reblock_blob

    def session_restore(self, blob, voice=0):
        self.calls.append(('session_restore', blob, voice))
        return 5

    def reblock_restore(self, blob):
        self.calls.append(('reblock_restore', blob))
        return 2

    def session_io_geometry(self, sid):
        return {'max_out': 6144}


def _drained_pipeline(engine, config, echo=False, index=42):
    from realtime_yukarin_b200.worker import RealtimePipeline
    p = RealtimePipeline.__new__(RealtimePipeline)
    p.config, p.engine, p._sid, p._rid = config, engine, 4, 1
    p._inflight, p._done, p._popped = collections.deque(), collections.deque(), []
    p._index_input = p._index_output = index
    p._echo, p._limiter = echo, True
    if echo:
        p._played = np.arange(37, dtype=np.float32) / 64
    return p


@pytest.mark.parametrize('echo', [False, True])
def test_pipeline_blob_packs_the_host_state(echo):
    from realtime_yukarin_b200.worker import RealtimePipeline, unpack_pipeline
    config = _config(input_scale=0.5, output_scale=2.0)
    sb, rb = _session_blob(), _reblock_blob(chunk=config.out_audio_chunk)
    src = _drained_pipeline(MoveEngine(sb, rb), config, echo=echo)
    blob = src.snapshot()
    d = describe_snapshot(blob)
    assert d['kind'] == 'pipeline' and [t for t, _ in d['sections']] == ['SESS', 'RBLK', 'PIPE'] + (['FARQ'] if echo else [])
    parts = unpack_pipeline(blob)
    assert parts['session'] == sb and parts['reblock'] == rb
    assert parts['host'] == {'index': 42, 'input_scale': 0.5, 'output_scale': 2.0, 'echo': echo, 'limiter': True}
    if echo:
        assert np.array_equal(parts['played'], src._played)
    dst_engine = MoveEngine()
    dst = RealtimePipeline.restore(blob, config, engine=dst_engine, voice=3, depth=4)
    assert dst_engine.calls == [('session_restore', sb, 3), ('reblock_restore', rb)]
    assert (dst._sid, dst._rid, dst.depth, dst._index_input, dst._index_output, dst._echo, dst._limiter) == (5, 2, 4, 42, 42, echo, True)
    assert len(dst._scratch) == 6144 and not dst._inflight and not dst._done and not dst._popped
    if echo:
        assert np.array_equal(dst._played, src._played)


def test_pipeline_snapshot_refuses_until_drained():
    from realtime_yukarin_b200.worker import Item
    config = _config()
    for field in ('_inflight', '_done', '_popped'):
        p = _drained_pipeline(MoveEngine(_session_blob(), _reblock_blob()), config)
        getattr(p, field).append(Item(None, 0))
        with pytest.raises(RuntimeError, match='drain'):
            p.snapshot()
        assert p.engine.calls == []


@pytest.mark.parametrize('change', [dict(buffer_time=0.2), dict(convert_extra_time=0.4), dict(input_silent_threshold=50.0),
                                    dict(input_rate=48000), dict(output_rate=48000), dict(output_silent_threshold=70.0),
                                    dict(input_scale=0.25), dict(output_scale=3.0), dict(vocoder_buffer_size=512)])
def test_pipeline_restore_refuses_another_configuration(change):
    from realtime_yukarin_b200.worker import RealtimePipeline
    config = _config()
    blob = _drained_pipeline(MoveEngine(_session_blob(), _reblock_blob(chunk=config.out_audio_chunk)), config).snapshot()
    dst_engine = MoveEngine()
    with pytest.raises(ValueError, match='another configuration'):
        RealtimePipeline.restore(blob, _config(**change), engine=dst_engine)
    assert dst_engine.calls == []
    RealtimePipeline.restore(blob, config, engine=dst_engine)       # the configuration it was taken with


def test_pipeline_restore_refuses_other_blobs():
    from realtime_yukarin_b200.worker import RealtimePipeline
    config = _config()
    blob = _drained_pipeline(MoveEngine(_session_blob(), _reblock_blob(chunk=config.out_audio_chunk)), config).snapshot()
    for bad in (_session_blob(), blob[:-5], snapshot.pack('pipeline', [('SESS', _session_blob())])):
        with pytest.raises(ValueError):
            RealtimePipeline.restore(bad, config, engine=MoveEngine())


# ---- run.py ---------------------------------------------------------------------------------------------------------------------
def test_run_state_options(tmp_path):
    from realtime_yukarin_b200 import run
    p = run.make_parser()
    a = p.parse_args(['--config_path', 'cfg.yaml', '--save_state', 'a.state', '--load_state', 'b.state'])
    assert a.save_state == Path('a.state') and a.load_state == Path('b.state')
    a = p.parse_args(['--config_path', 'cfg.yaml'])
    assert a.save_state is None and a.load_state is None
    for kw in (dict(denoise=0.0), dict(pitch=2.0), dict(echo_cancel=32), dict(limit=-1.0), dict(agc=-26.0), dict(follow_input_f0=200),
               dict(formant=1.0), dict(learn_noise=1.0)):
        with pytest.raises(ValueError, match='--load_state brings the stages'):
            run.run(Path('does-not-exist.yaml'), load_state=tmp_path / 'x.state', **kw)


def test_save_state_file_drains_then_writes(tmp_path):
    from realtime_yukarin_b200 import run

    class Pipe:
        def __init__(self):
            self.log = []

        def drain(self):
            self.log.append('drain')
            return []

        def snapshot(self):
            self.log.append('snapshot')
            return b'blob'

    pipe = Pipe()
    run.save_state_file(pipe, tmp_path / 's.state')
    assert pipe.log == ['drain', 'snapshot'] and (tmp_path / 's.state').read_bytes() == b'blob'


def test_describe_needs_no_engine():
    # the call is host-only: it runs wherever libryk.so loads, device or not
    lib = eng.load_library()
    blob = _session_blob()
    kind, version = ctypes.c_int(), ctypes.c_int()
    assert lib.ryk_snapshot_describe(blob, ctypes.c_size_t(len(blob)), ctypes.byref(kind), ctypes.byref(version), None, None, None, None, 0) == 3
    assert (kind.value, version.value) == (1, 1)


def test_pipeline_restore_prepares_crepe(monkeypatch):
    from realtime_yukarin_b200 import crepe
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.worker import RealtimePipeline
    calls = []
    monkeypatch.setattr(crepe, 'engine_with_model', lambda engine=None: calls.append(('model', engine)) or engine)
    monkeypatch.setattr(crepe, 'set_session_rate', lambda fs, engine: calls.append(('rate', fs, engine)))
    config = _config(extract_f0_mode=VocodeMode.CREPE)
    blob = _drained_pipeline(MoveEngine(_session_blob(f0_method=2), _reblock_blob(chunk=config.out_audio_chunk)), config).snapshot()
    dst_engine = MoveEngine()
    RealtimePipeline.restore(blob, config, engine=dst_engine)
    # the CREPE model and the session rate's taps are in place before the session is restored
    assert calls == [('model', dst_engine), ('rate', 24000, dst_engine)] and dst_engine.calls[0][0] == 'session_restore'
    calls.clear()
    world = _config()
    RealtimePipeline.restore(_drained_pipeline(MoveEngine(_session_blob(), _reblock_blob(chunk=world.out_audio_chunk)), world).snapshot(),
                             world, engine=MoveEngine())
    assert calls == []


def test_pipeline_snapshot_refuses_an_output_index_behind():
    p = _drained_pipeline(MoveEngine(_session_blob(), _reblock_blob()), _config())
    p._index_output -= 1
    with pytest.raises(RuntimeError, match='drain'):
        p.snapshot()


def _state_file(tmp_path, name, **conf):
    from realtime_yukarin_b200.worker import pack_pipeline
    path = tmp_path / name
    path.write_bytes(pack_pipeline(_session_blob(**conf), _reblock_blob(), {'index': 0, 'echo': False, 'limiter': False}, None))
    return path


def test_run_checks_end_of_run_options_against_the_state_file(tmp_path, monkeypatch):
    from realtime_yukarin_b200 import run
    monkeypatch.setattr(run.Config, 'from_yaml', lambda path: (_ for _ in ()).throw(RuntimeError('reached the config')))
    plain, measured = _state_file(tmp_path, 'plain.state'), _state_file(tmp_path, 'measured.state', denoise=1, f0_measure=1)
    with pytest.raises(ValueError, match='--save_noise_profile needs noise suppression'):
        run.run(Path('cfg.yaml'), load_state=plain, save_noise_profile=tmp_path / 'p.npy')
    with pytest.raises(ValueError, match='--measure_input_statistics needs f0 measuring'):
        run.run(Path('cfg.yaml'), load_state=plain, measure_input_statistics=tmp_path / 's.npy')
    # with the stages in the file both are accepted (the run then goes on to read the config)
    with pytest.raises(RuntimeError, match='reached the config'):
        run.run(Path('cfg.yaml'), load_state=measured, save_noise_profile=tmp_path / 'p.npy', measure_input_statistics=tmp_path / 's.npy')
    (tmp_path / 'bad.state').write_bytes(b'not a state file')
    with pytest.raises(ValueError):
        run.run(Path('cfg.yaml'), load_state=tmp_path / 'bad.state')


def test_run_writes_the_state_when_the_loop_ends_by_sigint(tmp_path, monkeypatch):
    """Ctrl-C ends a live loop with SystemExit from the signal handler; the state is still written."""
    from realtime_yukarin_b200 import run

    class Pipe:
        def __init__(self, *a, **kw):
            self.log = []

        def drain(self):
            self.log.append('drain')
            return []

        def snapshot(self):
            self.log.append('snapshot')
            return b'state'

        def close(self):
            self.log.append('close')

    class Converter:
        class acoustic_converter:
            class config:
                class dataset:
                    acoustic_param = None

    pipes = []
    monkeypatch.setattr(run.Config, 'from_yaml', lambda path: _config())
    monkeypatch.setattr(run.YukarinConverter, 'make_yukarin_converter', lambda **kw: Converter())
    monkeypatch.setattr(run, 'RealtimePipeline', lambda *a, **kw: pipes.append(Pipe()) or pipes[-1])
    monkeypatch.setattr(run.wave_io, 'load_wave', lambda *a, **kw: type('W', (), {'wave': np.zeros(4800, np.float32)}))

    def interrupted(*a, **kw):
        raise SystemExit(0)
    monkeypatch.setattr(run, 'audio_loop', interrupted)
    out = tmp_path / 'out.state'
    with pytest.raises(SystemExit):
        run.run(Path('cfg.yaml'), wav_in=tmp_path / 'x.wav', save_state=out)
    assert out.read_bytes() == b'state' and pipes[0].log == ['drain', 'snapshot', 'close']
