"""Host-side plugin API conformance (no GPU): the framing / indexing contract of the original project's
Stream + SegmentMethod layer, restated as known-answer tests, plus comparisons with what the original's own
code returned (stored under tests/golden/ by tests/golden/make_reference_golden.py)."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import dropin
from realtime_yukarin_b200.feature import AcousticFeature, AcousticFeatureWrapper, Wave
from realtime_yukarin_b200.params import AcousticParam, Param
from realtime_yukarin_b200.segment import (BaseSegmentMethod, FeatureWrapperSegmentMethod, Segment, WaveSegmentMethod)
from realtime_yukarin_b200.stream import BaseStream, ConvertStream, EncodeStream, StreamWrapper


class TextMethod(BaseSegmentMethod):
    def length(self, data):
        return len(data)

    def pad(self, width):
        return ' ' * width

    def pick(self, data, first, last):
        return data[first:last]

    def concat(self, datas):
        return ''.join(datas)


class TextStream(BaseStream):
    def process(self, start_time, time_length, extra_time):
        return self.fetch(start_time, time_length, extra_time)


def make_text_stream(rate=10):
    s = TextStream(TextMethod(rate), TextMethod(rate))
    s.add(start_time=0, data='a' * rate)
    s.add(start_time=1, data='b' * rate)
    return s


def test_segment_record():
    m = TextMethod(4)
    seg = Segment(start_time=1, data='xxxxxxxx', method=m)
    assert (seg.start_time, seg.data, seg.method) == (1, 'xxxxxxxx', m)
    assert seg.length == 8 and seg.time_length == 2.0 and seg.end_time == 3.0 and seg.sampling_rate == 4
    assert tuple(seg) == (1, 'xxxxxxxx', m)


def test_fetch_known_answers():            # base_stream.py:32-79 via tests/test_base_stream.py:65-93
    s = make_text_stream()
    assert s.fetch(0, 1, 0) == 'a' * 10
    assert s.fetch(0.5, 1, 0) == 'a' * 5 + 'b' * 5
    assert s.fetch(-0.5, 1, 0) == ' ' * 5 + 'a' * 5
    assert s.fetch(1.5, 1, 0) == 'b' * 5 + ' ' * 5
    assert s.fetch(0, 1, 0.3) == ' ' * 3 + 'a' * 10 + 'b' * 3
    assert s.fetch(0, 2, 0.3) == ' ' * 3 + 'a' * 10 + 'b' * 10 + ' ' * 3


def test_remove_keeps_segments_ending_after():   # tests/test_base_stream.py:47-63
    s = make_text_stream()
    s.add(start_time=2, data='c' * 10)
    for end, left in ((0, 3), (1, 2), (2, 1), (3, 0)):
        s.remove(end_time=end)
        assert len(s.stream) == left


def test_fetch_gap_between_segments_is_padded():
    s = TextStream(TextMethod(10), TextMethod(10))
    s.add(start_time=0, data='a' * 10)
    s.add(start_time=2, data='c' * 10)
    assert s.fetch(0.5, 2, 0) == 'a' * 5 + ' ' * 10 + 'c' * 5


class VocoderMock:
    acoustic_param = AcousticParam()


def test_encode_stream_wave_fetch():       # tests/test_encode_stream.py:34-85
    st = EncodeStream(vocoder=VocoderMock())
    sr = VocoderMock.acoustic_param.sampling_rate
    one, two = np.ones(sr, np.float32), np.ones(sr, np.float32) * 2
    st.add(0, one)
    st.add(1, two)
    np.testing.assert_equal(st.fetch(0, 1, 0), one)
    np.testing.assert_equal(st.fetch(0.5, 1, 0), np.concatenate([one[:sr // 2], two[:sr // 2]]))
    np.testing.assert_equal(st.fetch(-0.5, 1, 0), np.concatenate([np.zeros(sr // 2, np.float32), one[:sr // 2]]))
    np.testing.assert_equal(st.fetch(0, 2, 0.3), np.concatenate([np.zeros(sr // 10 * 3), one, two, np.zeros(sr // 10 * 3)]))
    assert st.out_segment_method.sampling_rate == 200


class AttrDict(dict):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.__dict__ = self


def _wrapper(values, lengths, sr=16000, rate=200):
    return AcousticFeatureWrapper(
        wave=Wave(np.concatenate([np.ones(round(t * sr), np.float32) * v for v, t in zip(values, lengths)]), sr),
        f0=np.concatenate([np.ones((round(t * rate), 1), np.float32) * v for v, t in zip(values, lengths)]))


def test_convert_stream_feature_wrapper_fetch():   # tests/test_convert_stream.py:19-104
    vc = AttrDict(
        acoustic_converter=AttrDict(config=AttrDict(dataset=AttrDict(acoustic_param=AcousticParam(sampling_rate=16000)))),
        super_resolution=AttrDict(config=AttrDict(dataset=AttrDict(param=Param()))),
        output_sampling_rate=24000)
    st = ConvertStream(voice_changer=vc)
    st.in_segment_method._keys = ['f0']
    st.add(0, _wrapper([1], [1]))
    st.add(1, _wrapper([2], [1]))
    assert st.fetch(0, 1, 0) == _wrapper([1], [1])
    assert st.fetch(0.5, 1, 0) == _wrapper([1, 2], [0.5, 0.5])
    assert st.fetch(-0.5, 1, 0) == _wrapper([0, 1], [0.5, 0.5])
    assert st.fetch(1.5, 1, 0) == _wrapper([2, 0], [0.5, 0.5])
    assert st.fetch(0, 1, 0.3) == _wrapper([0, 1, 2], [0.3, 1, 0.3])
    assert st.fetch(0, 2, 0.3) == _wrapper([0, 1, 2, 0], [0.3, 1, 1, 0.3])


def test_feature_wrapper_segment_method():          # tests/test_feature_wrapper_segment_method.py:17-70
    m = FeatureWrapperSegmentMethod(sampling_rate=100, wave_sampling_rate=10000, order=5, frame_period=10)
    seg = lambda v, t: _wrapper(v, t, sr=10000, rate=100)
    pad = m.pad(width=100)
    assert pad == seg([0], [1])
    assert pad.wave.wave.dtype == np.float32 and pad.f0.shape == (100, 1) and pad.mc.shape == (100, 6)
    full = seg([1], [1])
    assert m.pick(full, 0, 50) == seg([1], [0.5])
    assert m.pick(full, 50, 100) == seg([1], [0.5])
    m._keys = ['f0']
    assert m.concat([seg([0], [1]), seg([1], [1])]) == seg([0, 1], [1, 1])


def test_acoustic_feature_helpers():
    sizes = AcousticFeature.get_sizes(sampling_rate=24000, order=8)
    assert sizes == dict(f0=1, sp=513, ap=513, coded_ap=3, mc=9, voiced=1)
    s = AcousticFeature.silent(4, sizes, keys=['f0', 'ap', 'mc', 'voiced'])
    assert s.f0.shape == (4, 1) and s.voiced.dtype == bool and not s.voiced.any() and (s.ap == 0).all()
    assert set(s.__dict__) == {'f0', 'sp', 'ap', 'coded_ap', 'mc', 'voiced'}
    rebuilt = AcousticFeature(**s.__dict__)                       # __dict__ round-trips through the constructor
    assert rebuilt.mc is s.mc
    p = s.pick(1, -1, keys=['f0', 'mc'])
    assert len(p.f0) == 2
    c = AcousticFeature.concatenate([s, s], keys=['f0'])
    assert len(c.f0) == 8
    idx = s.indexing(np.array([True, False, True, False]))
    assert len(idx.f0) == 2 and len(idx.mc) == 2


@pytest.mark.parametrize('rate,T,extra', [(24000, 0.3, 0.0), (24000, 0.3, 0.1), (200, 0.3, 0.5), (200, 0.1, 0.5), (200, 1.0, 0.5), (200, 0.3, 0.05)])
def test_worker_drive_window_identity(rate, T, extra):
    """SURVEY A.9a: driven like the workers (add at extra + k T, process_next(T)), step k's window is
    exactly round((T + 2 extra) rate) items long and item i is input item k n - 2 e + i (0 where negative)."""
    class Ident(BaseStream):
        def process(self, start_time, time_length, extra_time):
            return self.fetch(start_time, time_length, extra_time)
    st = Ident(WaveSegmentMethod(rate), WaveSegmentMethod(rate))
    w = StreamWrapper(st, extra_time=extra)
    n, e = round(T * rate), round(extra * rate)
    start = extra
    for k in range(400):
        st.add(start_time=start, data=np.arange(k * n, (k + 1) * n, dtype=np.float32) + 1)
        start += T
        win = w.process_next(T)
        assert len(win) == round((T + 2 * extra) * rate)
        idx = k * n - 2 * e + np.arange(len(win))
        np.testing.assert_array_equal(win, np.where(idx >= 0, idx + 1, 0).astype(np.float32))
        if k % 50 == 49:
            st.remove(end_time=start - 3 * T - 4 * extra)


GOLDEN = Path(__file__).resolve().parent / 'golden'


def test_reference_check_py_runs_unmodified(small_models):
    """BASELINE config 1: the original project's own check.py (unmodified) driven through the drop-in aliases -- wav in,
    EncodeStream / ConvertStream / DecodeStream over 1 s pieces with extras (0, 1, 0), wav out -- with the GPU engine replaced by
    the oracle-backed stand-in, as tests/golden/make_reference_golden.py ran it: the wav it wrote (stored as a digest) must equal
    the same flow composed by hand from the oracle's functions."""
    from oracle import nets as onets
    from oracle import pipeline as opipe
    from oracle import world as W
    from realtime_yukarin_b200 import engine as eng_mod
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.models import F0Converter
    from tests.golden.make_reference_golden import check_digest
    try:
        N = 3
        x = synthetic.synthetic_speech(N + 0.4, stream=23)

        # the same flow by hand: per-piece analysis, convert windows of 1 + 1 + 1 s with silent padding outside the file, decode
        cfg = opipe.PathConfig()
        p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
        stats = F0Converter(small_models['input_statistics_path'], small_models['target_statistics_path']).stats()
        pieces = [x[i * 24000:(i + 1) * 24000] for i in range(N)]
        feats = [opipe.extract_features(w, cfg) for w in pieces]
        cat = {k: np.concatenate([f[k] for f in feats]) for k in ('f0', 'ap', 'mc', 'voiced')}
        wave_all = np.concatenate(pieces)
        T = 200
        silent_mc = np.zeros((1, cfg.order + 1), np.float32)
        silent_mc[0, 0] = opipe.SILENT_MC0
        win = opipe.StreamOracle._window
        synth = W.RealtimeSynthesizer(24000, 5.0, 1024, 1024)
        outs = []
        for i in range(N):
            first = (i - 1) * T
            wfeat = dict(f0=win(cat['f0'], first, 3 * T, 0.0), ap=win(cat['ap'], first, 3 * T, 0.0), mc=win(cat['mc'], first, 3 * T, silent_mc),
                         voiced=win(cat['voiced'], first, 3 * T, False))
            wwave = win(wave_all, first * cfg.hop, 3 * T * cfg.hop, 0.0)
            conv = opipe.convert_window(wwave, wfeat, cfg, p1, p2, stats, backend='torch')
            y = synth.decode(conv['f0'][T:-T].ravel().astype(np.float64), conv['sp'][T:-T], conv['ap'][T:-T])
            outs.append(np.nan_to_num(y, nan=0.0))
        ref = np.concatenate(outs).astype(np.float32)
        assert len(ref) > 0
        check_digest(dict(np.load(GOLDEN / 'reference_golden.npz')), 'check_py/out', ref, atol=1e-6 * max(1.0, float(np.abs(ref).max())))
    finally:
        eng_mod.set_default_engine(None)


REF_CONFIG = GOLDEN / 'reference_config.yaml'         # the original project's config.yaml


def test_config_reads_the_reference_yaml():
    """Config.from_yaml (config.py:44-71) on the original project's config.yaml: same fields, enum and derived chunk sizes."""
    from realtime_yukarin_b200.config import Config, VocodeMode
    c = Config.from_yaml(REF_CONFIG)
    assert c.input_rate == 24000 and c.output_rate == 24000 and c.frame_period == 5 and c.buffer_time == 1
    assert c.extract_f0_mode is VocodeMode.WORLD and c.vocoder_buffer_size == 1024
    assert (c.encode_extra_time, c.convert_extra_time, c.decode_extra_time) == (0.0, 0.5, 0.0)
    assert c.input_silent_threshold == 80 and c.output_silent_threshold == 80
    assert c.in_audio_chunk == 24000 and c.out_audio_chunk == 24000          # config.py:37-43
    assert isinstance(c.stage1_model_path, Path) and c.stage2_config_path.name == 'config.json'


def test_make_yukarin_converter_loads_both_stages(small_models):
    """YukarinConverter.make_yukarin_converter (converter/yukarin_converter.py:22-60): statistics, stage-1 and stage-2 models land
    in the engine (here the oracle-backed stand-in) and the converter exposes the objects VoiceChanger needs."""
    from realtime_yukarin_b200 import engine as eng_mod
    from realtime_yukarin_b200.converter import YukarinConverter
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    from tests.fake_engine import OracleEngine
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    eng_mod.set_default_engine(fake)
    try:
        conv = YukarinConverter.make_yukarin_converter(**{k: small_models[k] for k in (
            'input_statistics_path', 'target_statistics_path', 'stage1_model_path', 'stage1_config_path', 'stage2_model_path',
            'stage2_config_path')})
        assert conv.acoustic_converter.config.dataset.acoustic_param.sampling_rate == 24000
        assert fake.stats is not None and len(fake.stats) == 4           # log-f0 statistics reached the engine
        vc = VoiceChanger(super_resolution=conv.super_resolution, acoustic_converter=conv.acoustic_converter, threshold=80)
        assert vc.threshold == 80
    finally:
        eng_mod.set_default_engine(None)


def test_fetch_and_remove_differential_against_the_reference_classes():
    """Rows a1-a3 against the original project's BaseStream + a wave segment method: 300 seeded segment layouts (gaps, overlaps,
    touching segments), fetch windows and remove times, with the original's answers stored by tests/golden/make_reference_golden.py
    (segments left after remove, fetched arrays as sha256) -- this package's fetched arrays must be identical element for element."""
    from tests.golden.make_reference_golden import array_sha, run_fetch_case
    cases = json.loads((GOLDEN / 'reference_fetch_golden.json').read_text())
    assert len(cases) == 300
    for c in cases:
        c['layout'] = [tuple(x) for x in c['layout']]
        left, got = run_fetch_case(BaseStream, lambda rate: WaveSegmentMethod(sampling_rate=rate), c)
        assert left == c['left'], c
        assert len(got) == c['len'] and array_sha(got) == c['sha256'], c
