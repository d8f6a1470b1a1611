"""CREPE f0 front-end on the H100: the host mirror of `crepe.predict` / `crepe.predict_voicing` as the reference uses them in
realtime_voice_conversion/yukarin_wrapper/acoustic_feature_wrapper.py:65-80 (CrepeAcousticFeatureWrapper.extract_f0).

    t, f0, confidence, _ = crepe.predict(x, fs, viterbi=True, model_capacity='full', step_size=frame_period, verbose=0)
    voiced = (crepe.predict_voicing(confidence) == 1) | (confidence > 0.1);  f0[~voiced] = 0

The network, the Viterbi decoders and the local cents average run in libryk (csrc/crepe.cu); this module uploads a weight file, builds
the HMM log-probability tables exactly as crepe does (numpy), resamples to the model's 16 kHz with the package's polyphase resampler
and applies the voicing rule.  Weights: an npz {conv<l>.W (cout, cin, k), conv<l>.b, bn<l>.gamma/beta/mean/var (l = 1..6), dense.W
(360, 64 m), dense.b}; the trained CREPE weights are not redistributable with this repository -- point RYK_CREPE_MODEL (or
load_crepe_model) at a converted file.  No CPU fallback."""
import ctypes
import math
import os
from typing import Optional

import numpy

MODEL_SRATE = 16000
SESSION_RATE = 24000          # the streaming session's rate (config.yaml input_rate); its CREPE analysis resamples from it
CAPACITY = {'tiny': 4, 'small': 8, 'medium': 16, 'large': 24, 'full': 32}
_FILTERS = [32, 4, 4, 4, 8, 16]
_WIDTHS = [512, 64, 64, 64, 64, 64]

_loaded = {'engine': None, 'multiplier': None, 'rates': set()}


def pitch_hmm_tables():
    """crepe.to_viterbi_cents' HMM in the log domain: (log start, log transition [360][360], (log emission self, other))."""
    with numpy.errstate(divide='ignore'):
        xx, yy = numpy.meshgrid(range(360), range(360))
        transition = numpy.maximum(12 - abs(xx - yy), 0).astype(numpy.float64)
        transition = transition / numpy.sum(transition, axis=1)[:, None]
        self_emission = 0.1
        e_self = self_emission + (1 - self_emission) / 360
        e_other = (1 - self_emission) / 360
        return float(numpy.log(1.0 / 360)), numpy.ascontiguousarray(numpy.log(transition)), (float(numpy.log(e_self)), float(numpy.log(e_other)))


def load_crepe_model(path, engine=None) -> int:
    """Upload an npz weight file and the 24 kHz -> 16 kHz resampler taps that sessions in f0 method 'crepe' use; returns the
    capacity multiplier (4 tiny .. 32 full)."""
    from .engine import default_engine
    engine = engine or default_engine()
    w = numpy.load(path)
    mult = int(w['conv1.W'].shape[0]) // _FILTERS[0]
    if mult not in CAPACITY.values():
        raise ValueError(f'{path}: {w["conv1.W"].shape[0]} first-layer filters is not a CREPE capacity')
    lib, h = engine.lib, engine._h
    engine._check(lib.ryk_crepe_create(h, mult))
    f32 = lambda a: numpy.ascontiguousarray(a, dtype=numpy.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    for l in range(6):
        cin = 1 if l == 0 else _FILTERS[l - 1] * mult
        W = f32(w[f'conv{l + 1}.W'])
        if W.shape != (_FILTERS[l] * mult, cin, _WIDTHS[l]):
            raise ValueError(f'conv{l + 1}.W has shape {W.shape}')
        arrs = [W] + [f32(w[k]) for k in (f'conv{l + 1}.b', f'bn{l + 1}.gamma', f'bn{l + 1}.beta', f'bn{l + 1}.mean', f'bn{l + 1}.var')]
        engine._check(lib.ryk_crepe_set_conv(h, l, *[fp(a) for a in arrs]))
    Wd, bd = f32(w['dense.W']), f32(w['dense.b'])
    if Wd.shape != (360, 64 * mult):
        raise ValueError(f'dense.W has shape {Wd.shape}')
    engine._check(lib.ryk_crepe_set_dense(h, fp(Wd), fp(bd)))
    ls, lt, (es, eo) = pitch_hmm_tables()
    cents = numpy.ascontiguousarray(numpy.linspace(0, 7180, 360) + 1997.3794084376191)      # crepe's cents_mapping
    engine._check(lib.ryk_crepe_set_decoder_tables(h, lt.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                   cents.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.c_double(ls),
                                                   ctypes.c_double(es), ctypes.c_double(eo)))
    _loaded['engine'], _loaded['multiplier'], _loaded['rates'] = engine, mult, set()
    set_session_rate(SESSION_RATE, engine)
    return mult


def set_session_rate(fs: int, engine) -> None:
    """Upload the fs -> 16 kHz resampler taps (wave_io.resample_filter) that sessions at `fs` in f0 method 'crepe' need; once per
    loaded model and rate."""
    from . import wave_io
    fs = int(fs)
    if fs in _loaded.get('rates', ()):
        return
    g = math.gcd(fs, MODEL_SRATE)
    up, down = MODEL_SRATE // g, fs // g
    taps = numpy.ascontiguousarray(wave_io.resample_filter(up, down), dtype=numpy.float64)
    engine._check(engine.lib.ryk_crepe_set_resampler(engine._h, fs, up, down, taps.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(taps)))
    _loaded['rates'].add(fs)


def engine_with_model(engine=None):
    """`engine` (default: the process engine) with CREPE weights loaded, from RYK_CREPE_MODEL when none were loaded into it yet."""
    from .engine import default_engine
    engine = engine or default_engine()
    if _loaded['engine'] is not engine:
        path = os.environ.get('RYK_CREPE_MODEL')
        if not path:
            raise RuntimeError('no CREPE weights loaded: call realtime_yukarin_b200.crepe.load_crepe_model(path) or set RYK_CREPE_MODEL')
        load_crepe_model(path, engine)
    return engine


def predict(audio: numpy.ndarray, sr: int, step_size: float = 10.0, engine=None, details: bool = False):
    """crepe.predict(audio, sr, viterbi=True, step_size=...) -> (time, frequency, confidence, activation); details=True appends
    (voicing states, pitch-bin path)."""
    from . import wave_io
    engine = engine_with_model(engine)
    x = numpy.asarray(audio, dtype=numpy.float32)
    if x.ndim == 2:
        x = x.mean(1)
    x16 = wave_io.resample(x, int(sr), MODEL_SRATE, engine) if int(sr) != MODEL_SRATE else numpy.ascontiguousarray(x)
    F = int(engine.lib.ryk_crepe_num_frames(len(x16), ctypes.c_double(step_size)))
    f0 = numpy.zeros(F); conf = numpy.zeros(F, numpy.float32); voicing = numpy.zeros(F, numpy.int32)
    act = numpy.zeros((F, 360), numpy.float32); path = numpy.zeros(F, numpy.int32)
    engine._check(engine.lib.ryk_crepe_predict(
        engine._h, x16.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), len(x16), ctypes.c_double(step_size),
        f0.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), conf.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        voicing.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), act.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        path.ctypes.data_as(ctypes.POINTER(ctypes.c_int))))
    time = numpy.arange(F) * step_size / 1000.0
    if details:
        return time, f0, conf, act, voicing, path
    return time, f0, conf, act


def extract_f0(x: numpy.ndarray, fs: int, frame_period: float, engine=None):
    """CrepeAcousticFeatureWrapper.extract_f0 (acoustic_feature_wrapper.py:66-80): (f0, t)."""
    t, f0, conf, _, voicing, _ = predict(x, fs, step_size=frame_period, engine=engine, details=True)
    voiced = (voicing == 1) | (conf > 0.1)
    f0 = f0.copy()
    f0[~voiced] = 0
    return f0, t


def run_test_conv(engine, backend: int, x, W, bias) -> numpy.ndarray:
    """One CREPE-shaped conv layer on the device (ryk_crepe_test_conv): x [F][Win][Cin], W (Cout, Cin, k) -> ReLU(conv + bias)
    [F][Win - k + 1][Cout]; backend 0 = FP32 CUDA cores, 1 = 3xTF32 tensor cores."""
    x = numpy.ascontiguousarray(x, dtype=numpy.float32)
    W = numpy.ascontiguousarray(W, dtype=numpy.float32)
    bias = numpy.ascontiguousarray(bias, dtype=numpy.float32)
    F, Win, Cin = x.shape
    Cout, _, k = W.shape
    y = numpy.empty((F, Win - k + 1, Cout), numpy.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    engine._check(engine.lib.ryk_crepe_test_conv(engine._h, int(backend), F, Win, Cin, Cout, k, fp(x), fp(W), fp(bias), fp(y)))
    return y


def run_test_network(engine, backend: int, x16, step_size: float = 5.0, repeat: int = 0):
    """The loaded network and decoders on a 16 kHz signal with an explicit conv back-end (ryk_crepe_test_network):
    (activation [F][360], path [F], voicing [F], mean device ms per run over `repeat` timed runs or None)."""
    x16 = numpy.ascontiguousarray(x16, dtype=numpy.float32)
    F = int(engine.lib.ryk_crepe_num_frames(len(x16), ctypes.c_double(step_size)))
    act = numpy.zeros((F, 360), numpy.float32); path = numpy.zeros(F, numpy.int32); voicing = numpy.zeros(F, numpy.int32)
    ms = ctypes.c_float()
    engine._check(engine.lib.ryk_crepe_test_network(
        engine._h, int(backend), x16.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), len(x16), ctypes.c_double(step_size),
        act.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), path.ctypes.data_as(ctypes.POINTER(ctypes.c_int)),
        voicing.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), int(repeat), ctypes.byref(ms)))
    return act, path, voicing, (ms.value if repeat > 0 else None)
