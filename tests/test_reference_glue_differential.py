"""The original project's glue classes on top of this package's third-party replacements, pinned by stored outputs (CPU).

`realtime_voice_conversion/{stream,segment}/*.py`, `yukarin_wrapper/voice_changer.py`, `worker/*.py` and `config.py` of the
original (Hiroshiba/realtime-yukarin) are pure Python over `yukarin` / `become_yukarin` / the vocoder.  tests/golden/
make_reference_golden.py drove them over this package's replacements (the oracle-backed engine of tests/fake_engine.py) the way
the original's workers do and stored what they returned (tests/golden/reference_golden.npz); this package's own classes must give
the same on the same engine."""
import json
from pathlib import Path

import numpy as np
import pytest

from tests.golden.make_reference_golden import check_digest

GOLDEN = Path(__file__).resolve().parent / 'golden'
# the stored outputs come from torch-CPU float32 convolutions on another machine: its kernels may round differently
RTOL = 1e-5
STREAM_CASES = [(0.3, (0.0, 0.5, 0.0)), (0.1, (0.1, 0.2, 0.1))]
WORKER_T, WORKER_EXTRA = 0.3, (0.0, 0.5, 0.0)


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(GOLDEN / 'reference_golden.npz'))


def stream_tag(T, extra):
    return f'streams_T{T:g}_extra' + '_'.join(f'{e:g}' for e in extra)


def run_stream_chain(models, fake, T, extra, EncodeStream, ConvertStream, DecodeStream, StreamWrapper, VoiceChanger):
    """EncodeStream -> ConvertStream(VoiceChanger) -> DecodeStream over 1.5 s of synthetic speech in chunks of T seconds;
    per chunk: (encoded f0, converted f0, converted sp, decoded wave)"""
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    f0c = F0Converter(models['input_statistics_path'], models['target_statistics_path'])
    ac = AcousticConverter(create_from_json(models['stage1_config_path']), models['stage1_model_path'], f0_converter=f0c, engine=fake)
    sr = SuperResolution(create_sr_from_json(models['stage2_config_path']), models['stage2_model_path'], engine=fake)
    acp = create_from_json(models['stage1_config_path']).dataset.acoustic_param
    voc = RealtimeVocoder(acoustic_param=acp, out_sampling_rate=24000, extract_f0_mode=VocodeMode.WORLD)
    voc.create_synthesizer(buffer_size=1024, number_of_pointers=16)
    es, cs, ds = EncodeStream(vocoder=voc), ConvertStream(voice_changer=VoiceChanger(acoustic_converter=ac, super_resolution=sr, threshold=60)), DecodeStream(vocoder=voc)
    ws = [StreamWrapper(stream=es, extra_time=extra[0]), StreamWrapper(stream=cs, extra_time=extra[1]), StreamWrapper(stream=ds, extra_time=extra[2])]
    x = synthetic.synthetic_speech(1.5, 31)
    n = round(T * 24000)
    outs = []
    for k in range(len(x) // n):
        es.add(start_time=extra[0] + k * T, data=x[k * n:(k + 1) * n])
        f = ws[0].process_next(time_length=T)
        cs.add(start_time=extra[1] + k * T, data=f)
        c = ws[1].process_next(time_length=T)
        ds.add(start_time=extra[2] + k * T, data=c)
        y = ws[2].process_next(time_length=T)
        outs.append((np.asarray(f.f0).copy(), np.asarray(c.f0).copy(), np.asarray(c.sp).copy(), np.asarray(y.wave if hasattr(y, 'wave') else y).copy()))
    return outs


@pytest.mark.parametrize('T,extra', STREAM_CASES)
def test_reference_streams_and_voice_changer_over_our_replacements(small_models, golden, T, extra):
    from realtime_yukarin_b200 import engine as eng_mod
    from realtime_yukarin_b200 import stream as our_stream
    from realtime_yukarin_b200 import voice_changer as our_vc
    from tests.fake_engine import OracleEngine
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    eng_mod.set_default_engine(fake)
    try:
        got = run_stream_chain(small_models, fake, T, extra, our_stream.EncodeStream, our_stream.ConvertStream, our_stream.DecodeStream,
                               our_stream.StreamWrapper, our_vc.VoiceChanger)
        tag = stream_tag(T, extra)
        assert len(got) == int(golden[tag + '/chunks']) > 0
        for i, arrs in enumerate(got):
            for j, a in enumerate(arrs):
                check_digest(golden, f'{tag}/{i}/{j}', a, rtol=RTOL)
    finally:
        eng_mod.set_default_engine(None)


def librosa_module():
    """`librosa.stft` / `librosa.core.power_to_db` for the original's decode worker (decode_worker.py:56), written here in numpy
    (librosa 0.6/0.7 defaults: n_fft 2048, hop 512, periodic Hann, reflect-centred; ref 1, amin 1e-10, top_db 80).  Test harness only."""
    import types
    import scipy.signal as ss

    def stft(y, n_fft=2048, hop_length=None):
        hop = hop_length or n_fft // 4
        yp = np.pad(np.asarray(y, np.float64), n_fft // 2, mode='reflect')
        win = ss.get_window('hann', n_fft, fftbins=True)
        frames = 1 + len(y) // hop
        return np.stack([np.fft.rfft(yp[f * hop:f * hop + n_fft] * win) for f in range(frames)], 1)

    def power_to_db(S, ref=1.0, amin=1e-10, top_db=80.0):
        db = 10.0 * np.log10(np.maximum(amin, S)) - 10.0 * np.log10(np.maximum(amin, ref))
        return np.maximum(db, db.max() - top_db)

    lib = types.ModuleType('librosa'); lib.__path__ = []
    core = types.ModuleType('librosa.core')
    lib.stft, core.power_to_db, lib.core = stft, power_to_db, core
    return lib, core


def worker_models(models, fake):
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    f0c = F0Converter(models['input_statistics_path'], models['target_statistics_path'])
    ac = AcousticConverter(create_from_json(models['stage1_config_path']), models['stage1_model_path'], f0_converter=f0c, engine=fake)
    sr = SuperResolution(create_sr_from_json(models['stage2_config_path']), models['stage2_model_path'], engine=fake)
    acp = create_from_json(models['stage1_config_path']).dataset.acoustic_param
    return ac, sr, acp, RealtimeVocoder(acoustic_param=acp, out_sampling_rate=24000, extract_f0_mode=VocodeMode.WORLD)


def worker_setup(models, fake):
    """-> (config whose output threshold gates some chunks and keeps others, input audio, chunk count, chunks that pass ungated)"""
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import Item, RealtimePipeline
    T, extra = WORKER_T, WORKER_EXTRA
    x = synthetic.synthetic_speech(3.0, stream=37)
    x[int(1.2 * 24000):int(2.1 * 24000)] *= 1e-4
    n = round(T * 24000)
    K = len(x) // n
    acp = worker_models(models, fake)[2]

    def make_cfg(out_thr):
        return Config(input_device_name=None, output_device_name=None, input_rate=24000, output_rate=24000, frame_period=5.0, buffer_time=T,
                      extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0,
                      input_silent_threshold=60.0, output_silent_threshold=out_thr, encode_extra_time=extra[0],
                      convert_extra_time=extra[1], decode_extra_time=extra[2],
                      **{k: models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})

    # a threshold that gates some chunks and keeps others: powers of the ungated chunks, split at their widest gap
    lib, core = librosa_module()
    probe = RealtimePipeline(make_cfg(1e9), acoustic_param=acp, engine=fake, depth=1)
    powers = []
    for k in range(K):
        probe.put(Item(item=x[k * n:(k + 1) * n].copy(), index=k))
        it = probe.get()
        if it.item is not None:
            powers.append(float(core.power_to_db(np.abs(lib.stft(it.item)) ** 2).mean()))
    probe.close()
    ps = np.sort(np.asarray(powers))
    gi = int(np.argmax(np.diff(ps)))
    assert ps[gi + 1] - ps[gi] > 1e-3
    return make_cfg(-float(0.5 * (ps[gi] + ps[gi + 1]))), x, K, len(powers)


def test_reference_workers_over_our_replacements_match_realtime_pipeline(small_models, golden):
    """SURVEY 8(f) ranks 1 / 2 against the original's worker code: its encode_worker / convert_worker / decode_worker (each in a
    thread, queue.Queue standing in for multiprocessing.Queue) over this package's replacements, stored, versus
    worker.RealtimePipeline on the same engine: the same Items in the same order -- chunk played, or None (not enough samples
    yet / gated as silent)."""
    from realtime_yukarin_b200 import engine as eng_mod
    from realtime_yukarin_b200.worker import Item, RealtimePipeline
    from tests.fake_engine import OracleEngine
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    eng_mod.set_default_engine(fake)
    try:
        cfg, x, K, n_powers = worker_setup(small_models, fake)
        assert abs(cfg.output_silent_threshold - float(golden['workers/output_silent_threshold'])) <= RTOL * abs(cfg.output_silent_threshold)
        acp = worker_models(small_models, fake)[2]
        n = round(WORKER_T * 24000)
        pipe = RealtimePipeline(cfg, acoustic_param=acp, engine=fake, depth=1)
        ours = []
        for k in range(K):
            pipe.put(Item(item=x[k * n:(k + 1) * n].copy(), index=k))
            ours.append(pipe.get())
        pipe.close()
        assert list(golden['workers/index']) == [it.index for it in ours] == list(range(K))
        played = 0
        for k, (ref_played, b) in enumerate(zip(golden['workers/played'], ours)):
            assert bool(ref_played) == (b.item is not None), k
            if b.item is not None:
                played += 1
                assert len(b.item) == cfg.out_audio_chunk
                check_digest(golden, f'workers/{k}', b.item, atol=1e-9, rtol=RTOL)
        assert 0 < played < n_powers                     # the gate kept some chunks and dropped others, identically on both sides
    finally:
        eng_mod.set_default_engine(None)


def test_reference_converter_and_config_modules_over_our_replacements():
    """The original's config.py reads its config.yaml (stored) into the values in reference_config_fields.json; this package's
    Config reads the same values from the same file."""
    from realtime_yukarin_b200 import config as our_config
    want = json.loads((GOLDEN / 'reference_config_fields.json').read_text())
    b = our_config.Config.from_yaml(GOLDEN / 'reference_config.yaml')
    for name in set(want) - {'in_audio_chunk', 'out_audio_chunk'}:
        vb = getattr(b, name)
        vb = vb.value if hasattr(vb, 'value') else vb
        assert (str(vb) if isinstance(vb, Path) else vb) == want[name], name
    assert b.in_audio_chunk == want['in_audio_chunk'] and b.out_audio_chunk == want['out_audio_chunk']
