"""CREPE f0 mode on the H100 (csrc/crepe.cu, realtime_yukarin_b200/crepe.py) against the restatement in oracle/crepe.py, with seeded
synthetic weights: (1) the network -- activations within FP32 accumulation tolerance; (2) the decoders -- Viterbi pitch path, local
cents average and the voicing HMM applied by the oracle to the SAME activations must reproduce the device decisions exactly;
(3) end to end through CrepeAcousticFeatureWrapper / Vocoder(extract_f0_mode=CREPE)."""
import numpy as np
import pytest
from scipy.signal import resample_poly

from oracle import crepe as oc
from realtime_yukarin_b200 import crepe as pcrepe
from realtime_yukarin_b200 import synthetic

from .test_gpu_parity import CFG, _speech

pytestmark = pytest.mark.gpu


def _x16(seconds, stream):
    x = _speech(seconds, stream)
    return x, resample_poly(x.astype(np.float64), 2, 3).astype(np.float32)


@pytest.mark.parametrize('capacity,seconds,bias_shift', [('tiny', 0.9, 0.0), ('tiny', 0.9, -2.0), ('tiny', 0.9, -4.5), ('full', 0.3, 0.0)])
def test_crepe_network_and_decoders_match_oracle(engine, tmp_path, capacity, seconds, bias_shift):
    w = synthetic.make_crepe_params(3, capacity)
    w['dense.b'] = (w['dense.b'] + bias_shift).astype(np.float32)        # bias_shift -2: confidences around 0.5; -4.5: below 0.1 (unvoiced state, f0 zeroed)
    path = tmp_path / 'crepe.npz'
    np.savez(path, **w)
    assert pcrepe.load_crepe_model(path, engine) == pcrepe.CAPACITY[capacity]
    _, x16 = _x16(seconds, 21)
    t, f0, conf, act, voicing, ppath = pcrepe.predict(x16, 16000, step_size=5.0, engine=engine, details=True)
    act_ref = oc.get_activation(x16, w, 5.0)
    assert act.shape == act_ref.shape
    err = float(np.abs(act - act_ref).max())
    print(f'crepe {capacity}: {act.shape[0]} frames, activation max |err| {err:.2e}, confidence range {conf.min():.3f}..{conf.max():.3f}')
    assert err < 5e-4
    assert np.allclose(conf, act.max(1))
    # decoders on the device's own activations
    cents, path_ref = oc.to_viterbi_cents(act)
    assert np.array_equal(ppath, path_ref)
    assert np.allclose(f0, 10 * 2 ** (cents / 1200), rtol=1e-9)
    v_ref = oc.predict_voicing(conf)
    assert np.array_equal(voicing, v_ref)
    print(f'   voicing states: {int(voicing.sum())} voiced of {len(voicing)}')
    if bias_shift <= -4:
        assert voicing.sum() == 0
    assert np.allclose(t, np.arange(len(f0)) * 0.005)
    # end to end against the oracle's own activations: the decisions agree wherever the oracle's arg-max margin is not marginal
    f0_ref, _ = oc.extract_f0(x16, w, 5.0)
    f0_dev, _ = pcrepe.extract_f0(x16, 16000, 5.0, engine=engine)
    same = np.isclose(f0_dev, f0_ref, rtol=1e-6)
    print(f'   end to end: {int(same.sum())} of {len(same)} frames identical')
    assert same.mean() > 0.9


def test_crepe_mode_through_the_vocoder(engine, tmp_path):
    from realtime_yukarin_b200.config import VocodeMode
    from realtime_yukarin_b200.feature import Wave
    from realtime_yukarin_b200.params import AcousticParam
    from realtime_yukarin_b200.vocoder import Vocoder
    path = synthetic.write_crepe_model(tmp_path, seed=5, capacity='tiny')
    pcrepe.load_crepe_model(path, engine)
    x = _speech(0.6, 9)
    voc = Vocoder(AcousticParam(), out_sampling_rate=24000, extract_f0_mode=VocodeMode.CREPE)
    feat = voc.encode(Wave(wave=x, sampling_rate=24000))
    f0, t = pcrepe.extract_f0(x, 24000, 5.0, engine=engine)
    n = len(x) // CFG.hop
    assert feat.f0.shape == (n, 1) and feat.sp.shape == (n, 513)
    assert np.allclose(feat.f0.ravel(), f0[:n].astype(np.float32))
    assert np.array_equal(feat.voiced.ravel(), f0[:n] != 0)
    assert np.all(np.isfinite(feat.sp)) and np.all(feat.sp > 0)
