"""The signals of tests/gated_speech.py do what tests/test_gpu_silence_gate_paths.py needs of them, and the host classes handle a
partial mask -- all on the CPU, against the oracle.

  * every window case reaches its count with its margin, the counts are exactly {1, 127, 128, 129, 255, 256, 257, 260}, 'tail' and
    'comb' masks are far from the identity, and the quiet part is effective again at 80 dB;
  * the stream with pauses walks the stage-1 buckets 1, 2 and 3, every one of a session's six stage-1 graph copies (step % 6) in more
    than one of them;
  * VoiceChanger's staged route (separate_effective -> convert -> combine_silent) over the oracle-backed engine stand-in equals
    oracle.pipeline.convert_window on a 'comb' window and on a window without any effective frame (threshold 0);
  * EncodeStream / ConvertStream / DecodeStream reproduce the oracle's closed-form stream on the stream with pauses.
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import engine as eng_mod
from tests import gated_speech as gs
from tests.fake_engine import OracleEngine

CFG = gs.CFG
TW = 260


@pytest.mark.parametrize('pattern,target,zeros', gs.WINDOW_CASES)
def test_window_cases_reach_their_count(pattern, target, zeros):
    wave, mask = gs.window_with_count(target, TW, 60.0, pattern, zeros)
    assert len(wave) == TW * gs.HOP and wave.dtype == np.float32
    assert int(mask.sum()) == target and gs.mask_margin(wave, TW, 60.0) >= gs.MIN_MARGIN_DB
    index = np.flatnonzero(mask)
    if pattern == 'head':
        assert np.array_equal(index, np.arange(target))
    elif pattern == 'tail':
        assert np.array_equal(index, np.arange(TW - target, TW))
    else:
        lag = index - np.arange(target)                     # how far each effective frame's rank falls behind its index
        assert len(np.unique(lag)) >= 4 and lag[0] == 0, np.unique(lag)
    if zeros:
        assert (wave[np.repeat(~mask, gs.HOP)] == 0).any()
        assert gs.count_effective(wave, TW, 80.0) == target     # digital silence stays gated at any threshold
    else:
        assert gs.count_effective(wave, TW, 80.0) == TW and gs.mask_margin(wave, TW, 80.0) >= gs.MIN_MARGIN_DB
    assert gs.count_effective(wave, TW, None) == TW
    assert gs.count_effective(wave, TW, 0.0) == 0           # threshold 0: not even the loudest frame is above itself


def test_counts_cover_the_bucket_edges():
    full = gs.window_with_count(TW, TW, 60.0, 'head')[1]
    assert full.all()
    wave, thr, mask = gs.peak_window(TW)
    assert int(mask.sum()) == 1 and 0 < thr < 1
    assert {t for _, t, _ in gs.WINDOW_CASES} | {1, TW} == {1, 127, 128, 129, 255, 256, 257, 260}
    # the padded length the oracle's 'minimum' pad gives, and the bucket it selects
    for t, tp in ((1, 128), (127, 128), (128, 256), (129, 256), (255, 256), (256, 384), (257, 384), (260, 384)):
        assert t + 128 - t % 128 == tp


@pytest.mark.parametrize('zeros', [False, True])
def test_stream_with_pauses_walks_the_buckets(zeros):
    x = gs.stream_with_pauses(zeros=zeros)
    steps = len(x) // round(0.3 * gs.FS)
    assert steps >= 30
    rows = gs.step_counts(x, steps, 60.0)
    buckets = [b for _, b, _ in rows]
    assert min(m for _, _, m in rows) >= gs.MIN_MARGIN_DB
    assert set(buckets) == {1, 2, 3}
    for steps_used in (24, 30):
        for j in range(6):
            assert len(set(buckets[j:steps_used:6])) >= 2, (steps_used, j, buckets[j:steps_used:6])
    assert set(buckets[4:24]) == {1, 2, 3}                  # after the start-up steps, whose window still holds the zeros before the stream
    # the counts are not all multiples of the chunk: pauses begin and end inside chunks
    assert len({c % 60 for c, _, _ in rows}) > 6


def _host_classes(paths, fake):
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    ac = AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=fake)
    sr = SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=fake)
    return ac, sr, f0c


@pytest.mark.parametrize('threshold,target', [(60.0, 128), (0.0, 0)])
def test_staged_voice_changer_on_a_partial_mask(small_models, threshold, target):
    from realtime_yukarin_b200.feature import AcousticFeatureWrapper, Wave
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    eng_mod.set_default_engine(fake)
    try:
        ac, sr, f0c = _host_classes(small_models, fake)
        p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
        wave, _ = gs.window_with_count(128, TW, 60.0, 'comb')
        enc = opipe.extract_features(wave, CFG)
        ref = opipe.convert_window(wave, enc, CFG, p1, p2, f0c.stats(), backend='torch', threshold_db=threshold)
        eff = ref['effective']
        assert int(eff.sum()) == target
        fw = AcousticFeatureWrapper(wave=Wave(wave, CFG.fs), f0=enc['f0'], ap=enc['ap'], mc=enc['mc'], voiced=enc['voiced'])
        out = VoiceChanger(ac, sr, threshold=threshold).convert_from_acoustic_feature(fw)
        assert np.array_equal(out.voiced.ravel(), ref['voiced'].ravel())
        assert np.array_equal(out.f0.ravel(), ref['f0'].ravel())
        assert np.array_equal(out.ap, ref['ap'])
        assert np.array_equal(out.mc, ref['mc'])
        assert np.allclose(out.sp, ref['sp'], rtol=1e-5)
        # the silent template on every gated frame
        assert (out.mc[~eff, 0] == np.float32(opipe.SILENT_MC0)).all() and not out.mc[~eff, 1:].any()
        assert not out.ap[~eff].any() and not out.f0[~eff].any() and not out.voiced[~eff].any()
        assert enc['voiced'][~eff].any()                    # the gate disagrees with the voicing: the template, not the input, wins
    finally:
        eng_mod.set_default_engine(None)


def test_stream_classes_on_the_stream_with_pauses(small_models):
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.params import create_from_json
    from realtime_yukarin_b200.stream import ConvertStream, DecodeStream, EncodeStream, StreamWrapper
    from realtime_yukarin_b200.vocoder import RealtimeVocoder
    from realtime_yukarin_b200.voice_changer import VoiceChanger
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    eng_mod.set_default_engine(fake)
    try:
        ac, sr, f0c = _host_classes(small_models, fake)
        acp = create_from_json(small_models['stage1_config_path']).dataset.acoustic_param
        voc = RealtimeVocoder(acoustic_param=acp, out_sampling_rate=24000, extract_f0_mode=VocodeMode.WORLD)
        voc.create_synthesizer(buffer_size=1024, number_of_pointers=16)
        T, extra, steps = 0.3, (0.0, 0.5, 0.0), 14
        es, cs, ds = EncodeStream(voc), ConvertStream(VoiceChanger(ac, sr, threshold=60)), DecodeStream(voc)
        ws = [StreamWrapper(es, extra[0]), StreamWrapper(cs, extra[1]), StreamWrapper(ds, extra[2])]
        p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        x = gs.stream_with_pauses()
        assert {b for _, b, _ in gs.step_counts(x, steps, 60.0)} == {1, 2, 3}
        n = round(T * 24000)
        for k in range(steps):
            chunk = x[k * n:(k + 1) * n]
            es.add(start_time=extra[0] + k * T, data=chunk)
            f = ws[0].process_next(T)
            cs.add(start_time=extra[1] + k * T, data=f)
            c = ws[1].process_next(T)
            ds.add(start_time=extra[2] + k * T, data=c)
            y = ws[2].process_next(T)
            r = orc.push(chunk)
            assert np.array_equal(c.f0, orc.last['converted']['f0']), k
            assert np.array_equal(c.ap, orc.last['converted']['ap']), k
            assert np.allclose(c.sp, orc.last['converted']['sp'], rtol=1e-5), k
            assert len(y) == len(r), (k, len(y), len(r))
            assert np.allclose(y, r, atol=1e-9), k
    finally:
        eng_mod.set_default_engine(None)
