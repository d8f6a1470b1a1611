"""RealtimePipeline.set_voice on the CPU, over an oracle-backed session stand-in that records the order of its calls.

  * set_voice finishes every chunk in flight before it switches, and the switch lands before the next chunk is submitted;
  * the outputs keep their order through the switch and equal the switching oracle (StreamOracle with stage1 / stage2 / f0_stats
    swapped between pushes), re-blocked as the pipeline re-blocks them;
  * the switching oracle is bitwise the old voice's oracle before the switch and differs from it after.
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic
from tests.fake_engine import OracleEngine

K, KS = 7, 3                    # chunks, the chunk from which the stream converts into the second voice
DEFAULT_STATS = (float(np.log(150.0)), 0.2, float(np.log(250.0)), 0.2)     # the stand-in's voice 0 (see fake_engine.session_create)


class SwitchingEngine(OracleEngine):
    """OracleEngine with voices and ryk_session_set_voice's rules: every submitted chunk collected, the oracle's nets and f0 statistics
    swapped for the next push.  Its device is never done when polled, so chunks stay in flight until the pipeline collects them."""

    def __init__(self, stage1_npz, stage2_npz):
        super().__init__(stage1_npz, stage2_npz)
        self.voices = {0: (self.p1, self.p2, DEFAULT_STATS)}
        self.calls = []

    def add_voice(self, paths):
        from realtime_yukarin_b200.models import F0Converter
        vid = max(self.voices) + 1
        stats = F0Converter(paths['input_statistics_path'], paths['target_statistics_path']).stats()
        self.voices[vid] = (onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path']), stats)
        return vid

    def session_poll(self, sid, ticket):
        return False

    def reblock_poll(self, rid, ticket):
        return False

    def session_submit(self, sid, wave):
        ticket = super().session_submit(sid, wave)
        self.calls.append(('submit', ticket))
        return ticket

    def session_collect(self, sid, ticket, out):
        self.calls.append(('collect', ticket))
        return super().session_collect(sid, ticket, out)

    def session_set_voice(self, sid, voice):
        S = self.sessions[sid]
        assert not S['out'], 'collect every submitted chunk before switching the voice'
        orc = S['orc']
        orc.stage1, orc.stage2, orc.f0_stats = self.voices[voice]
        self.calls.append(('set_voice', voice))


@pytest.fixture(scope='module')
def second_voice(tmp_path_factory):
    return synthetic.write_synthetic_models(tmp_path_factory.mktemp('switch_voice'), seed=57, base1=16, base2=16)


def _config(small_models):
    from realtime_yukarin_b200.config import Config, VocodeMode
    return Config(input_device_name=None, output_device_name=None, input_rate=24000, output_rate=24000, frame_period=5.0, buffer_time=0.3,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0,
                  **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path', 'stage1_config_path',
                                                  'stage2_model_path', 'stage2_config_path')})


def _oracle(engine, voice):
    p1, p2, stats = engine.voices[voice]
    return opipe.StreamOracle(opipe.PathConfig(threshold_db=60.0), p1, p2, stats, buffer_time=0.3, extra=(0.0, 0.5, 0.0), backend='torch')


def test_set_voice_drains_then_switches(small_models, second_voice):
    from realtime_yukarin_b200.worker import Item, RealtimePipeline
    fake = SwitchingEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    vb = fake.add_voice(second_voice)
    cfg = _config(small_models)
    n = cfg.in_audio_chunk
    x = synthetic.synthetic_speech((K + 1) * 0.3, stream=19)
    chunks = [np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32) for k in range(K)]

    # the switching oracle, the first voice's and the second voice's, and the switching one re-blocked as the pipeline re-blocks
    switching, only_a, only_b = _oracle(fake, 0), _oracle(fake, 0), _oracle(fake, vb)
    rb = opipe.OutputReblockOracle(cfg.out_audio_chunk, 80.0)
    sw, a, b, expected = [], [], [], []
    for k, c in enumerate(chunks):
        if k == KS:
            switching.stage1, switching.stage2, switching.f0_stats = fake.voices[vb]
        sw.append(switching.push(c))
        a.append(only_a.push(c))
        b.append(only_b.push(c))
        expected.append(rb.push(sw[-1])[1])
    assert all(np.array_equal(sw[k], a[k]) for k in range(KS))
    after = np.concatenate(sw[KS:])
    assert not np.array_equal(after, np.concatenate(a[KS:])) and not np.array_equal(after, np.concatenate(b[KS:]))

    pipe = RealtimePipeline(cfg, engine=fake, depth=3)
    try:
        for k, c in enumerate(chunks):
            if k == KS:
                pipe.set_voice(vb)
            pipe.put(Item(item=c, index=k))
        got = [pipe.get() for _ in range(K)]
    finally:
        pipe.close()
    # drain, then switch, then the next chunk
    i = fake.calls.index(('set_voice', vb))
    assert sorted(t for op, t in fake.calls[:i] if op == 'collect') == list(range(KS))
    assert sorted(t for op, t in fake.calls[:i] if op == 'submit') == list(range(KS))
    assert fake.calls[i + 1] == ('submit', KS)
    # order and values
    assert [it.index for it in got] == list(range(K))
    for k, it in enumerate(got):
        assert (it.item is None) == (expected[k] is None), k
        if it.item is not None:
            assert np.array_equal(it.item, expected[k]), k


def test_set_voice_refused_with_chunks_in_flight_by_the_stand_in(small_models, second_voice):
    """The stand-in keeps the library's rule, so the ordering test above would fail if set_voice did not drain first."""
    fake = SwitchingEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    vb = fake.add_voice(second_voice)
    from realtime_yukarin_b200.engine import SessionConfig
    sid = fake.session_create(SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8,
                                            alpha=0.466, buffer_time=0.3, encode_extra_time=0.0, convert_extra_time=0.5,
                                            decode_extra_time=0.0, threshold_db=60.0, vocoder_buffer_size=1024))
    fake.session_submit(sid, np.zeros(7200, np.float32))
    with pytest.raises(AssertionError):
        fake.session_set_voice(sid, vb)
