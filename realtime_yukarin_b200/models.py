"""Model-side call surface kept from the reference's third-party imports, re-implemented on libryk:

  yukarin.f0_converter.F0Converter          (check.py:46-49, converter/yukarin_converter.py:35-38)
  yukarin.AcousticConverter                 (check.py:54-59; used by voice_changer.py:27-38)
  become_yukarin.SuperResolution            (check.py:60-63; used by voice_changer.py:41)

Model files keep the Chainer `save_npz` layout (`encoder/c1/c/W`, `encoder/c1/batchnorm/avg_var`, ...)
so that a real predictor.npz loads unchanged; eval-mode BatchNorm (eps 2e-5) and the conv bias are
folded into one per-channel scale/shift on load, weights are uploaded once and repacked on the GPU.
Statistics `.npy` files are pickled dicts {'mean', 'var'} of log-f0, as upstream writes them.
"""
from pathlib import Path
from typing import Dict, Optional, Tuple

import numpy

from .engine import Engine, default_engine
from .feature import SILENT_MC0, AcousticFeature
from .params import Config, SRConfig
from .world_consts import cheaptrick_fft_size

BN_EPS = 2e-5


def load_npz(path) -> Dict[str, numpy.ndarray]:
    with numpy.load(str(path), allow_pickle=False) as z:
        d = {k: z[k] for k in z.files}
    # strip an optional common prefix such as 'predictor/'
    if d and all(k.startswith('predictor/') for k in d):
        d = {k[len('predictor/'):]: v for k, v in d.items()}
    return d


def fold_layers(params: Dict[str, numpy.ndarray]):
    """-> list of 16 (W, scale, shift) in forward order: encoder c0..c7, decoder c0..c7."""
    layers = []
    for part in ('encoder', 'decoder'):
        for i in range(8):
            plain = (part == 'encoder' and i == 0) or (part == 'decoder' and i == 7)
            if plain:
                W = params[f'{part}/c{i}/W']
                b = params.get(f'{part}/c{i}/b')
                cout = W.shape[0]
                scale = numpy.ones(cout, numpy.float32)
                shift = numpy.zeros(cout, numpy.float32) if b is None else b.astype(numpy.float32)
            else:
                W = params[f'{part}/c{i}/c/W']
                b = params.get(f'{part}/c{i}/c/b')
                cout = W.shape[0] if part == 'encoder' else W.shape[1]
                bn = f'{part}/c{i}/batchnorm'
                if f'{bn}/gamma' in params:
                    gamma, beta = params[f'{bn}/gamma'], params[f'{bn}/beta']
                    mean, var = params[f'{bn}/avg_mean'], params[f'{bn}/avg_var']
                    scale = (gamma / numpy.sqrt(var + BN_EPS)).astype(numpy.float32)
                    bias = numpy.zeros(cout, numpy.float32) if b is None else b
                    shift = ((bias - mean) * scale + beta).astype(numpy.float32)
                else:
                    scale = numpy.ones(cout, numpy.float32)
                    shift = numpy.zeros(cout, numpy.float32) if b is None else b.astype(numpy.float32)
            layers.append((numpy.ascontiguousarray(W, numpy.float32), scale, shift))
    return layers


def upload_unet(engine: Engine, stage: int, params: Dict[str, numpy.ndarray], voice: int = 0):
    layers = fold_layers(params)
    w0 = layers[0][0]
    in_ch, base = w0.shape[1], w0.shape[0]
    out_ch = layers[15][0].shape[0]
    kw = {'voice': voice} if voice else {}          # voice 0: the calls existing callers make
    engine.model_create(stage, in_ch, out_ch, base, **kw)
    for i, (W, scale, shift) in enumerate(layers):
        tr, cin, cout, k = engine.model_layer_shape(stage, i, **kw)
        expect = (cin, cout) if tr else (cout, cin)
        if tuple(W.shape[:2]) != expect or W.shape[-1] != k:
            raise ValueError(f'stage {stage} layer {i}: weight shape {W.shape} does not match the U-Net topology '
                             f'(transposed={tr}, cin={cin}, cout={cout}, k={k})')
        engine.model_set_layer(stage, i, W, scale, shift, **kw)
    return in_ch, out_ch, base


def load_voice(engine: Engine, voice: int, *, stage1_model_path, stage2_model_path, input_statistics_path, target_statistics_path,
               feature_stats=None) -> None:
    """Load one target voice into `engine` (voice 0, or an id from engine.voice_create()): both U-Nets, the stage-1 feature
    statistics and the log-f0 statistics, with the same model-file rules as AcousticConverter / SuperResolution / F0Converter.
    Sessions created with engine.session_create(cfg, voice=voice) then convert into it."""
    params = load_npz(stage1_model_path)
    in_ch, out_ch, _ = upload_unet(engine, 1, params, voice=voice)
    stats = load_stage1_stats(params, stage1_model_path, in_ch, out_ch, feature_stats)
    upload_unet(engine, 2, load_npz(stage2_model_path), voice=voice)
    engine.stage1_set_stats(*stats, voice=voice)
    engine.f0_set_stats(*F0Converter(input_statistics_path, target_statistics_path).stats(), voice=voice)


class F0Converter(object):
    def __init__(self, input_statistics: Path, target_statistics: Path) -> None:
        def _load(p):
            d = numpy.load(str(p), allow_pickle=True)
            d = d.item() if isinstance(d, numpy.ndarray) else d
            return float(d['mean']), float(d['var'])
        self.input_mean, self.input_var = _load(input_statistics)
        self.target_mean, self.target_var = _load(target_statistics)

    def stats(self) -> Tuple[float, float, float, float]:
        return self.input_mean, float(numpy.sqrt(self.input_var)), self.target_mean, float(numpy.sqrt(self.target_var))

    def convert(self, in_f0: numpy.ndarray, engine: Optional[Engine] = None) -> numpy.ndarray:
        engine = engine or default_engine()
        engine.f0_set_stats(*self.stats())
        f0 = numpy.asarray(in_f0, dtype=numpy.float32)
        return engine.f0_convert(f0.ravel(), f0.ravel() != 0).reshape(f0.shape)


def write_f0_statistics(path, mean: float, var: float) -> None:
    """Write a log-f0 statistics file as upstream's training scripts do and F0Converter reads: a pickled dict {'mean', 'var'} in a
    `.npy` (numpy.save of a dict), e.g. from engine.session_f0_measured -> (n, mean, std): var = std ** 2."""
    mean, var = float(mean), float(var)
    if not (numpy.isfinite(mean) and numpy.isfinite(var) and var > 0):
        raise ValueError(f'log-f0 statistics need a finite mean and a positive variance, got mean {mean}, var {var}')
    with open(str(path), 'wb') as f:             # (a file object: numpy.save would append '.npy' to another suffix)
        numpy.save(f, numpy.array({'mean': mean, 'var': var}, dtype=object), allow_pickle=True)


STATS_KEYS = ('stats/in_mean', 'stats/in_std', 'stats/out_mean', 'stats/out_std')


def load_stage1_stats(params: Dict[str, numpy.ndarray], model_path, in_ch: int, out_ch: int, feature_stats=None):
    """Mel-cepstrum normalisation of stage 1 (SURVEY A.6 "input mean/var ... target mean/var", DECIDE 8).  Sources, in order:
      1. `feature_stats` = (in_mean, in_std, out_mean, out_std) arrays or a path to an .npz holding the `stats/*` keys,
      2. `stats/*` keys inside the model file (what synthetic.py writes),
      3. `<model dir>/stats.npz` next to predictor.npz.
    A bare Chainer predictor.npz has none of them: converting un-normalised features would run without any error and give
    garbage, so that case RAISES instead of silently falling back to identity.  Pass feature_stats='identity' to opt in."""
    def from_mapping(m):
        return tuple(numpy.asarray(m[k], numpy.float32) for k in STATS_KEYS)
    if isinstance(feature_stats, str) and feature_stats == 'identity':
        st = (numpy.zeros(in_ch, numpy.float32), numpy.ones(in_ch, numpy.float32), numpy.zeros(out_ch, numpy.float32), numpy.ones(out_ch, numpy.float32))
    elif isinstance(feature_stats, (str, Path)):
        with numpy.load(str(feature_stats), allow_pickle=False) as z:
            st = from_mapping(z)
    elif feature_stats is not None:
        st = tuple(numpy.asarray(a, numpy.float32) for a in feature_stats)
    elif all(k in params for k in STATS_KEYS):
        st = from_mapping(params)
    elif (Path(model_path).parent / 'stats.npz').exists():
        with numpy.load(str(Path(model_path).parent / 'stats.npz'), allow_pickle=False) as z:
            st = from_mapping(z)
    else:
        raise ValueError(
            f'{model_path}: no stage-1 feature normalisation statistics (keys {STATS_KEYS} in the model file, a stats.npz next to '
            "it, or feature_stats=...). Upstream yukarin keeps them outside predictor.npz; pass feature_stats='identity' only if the "
            'model was really trained on un-normalised mel-cepstra.')
    if [len(a) for a in st] != [in_ch, in_ch, out_ch, out_ch]:
        raise ValueError(f'stage-1 statistics have lengths {[len(a) for a in st]}, the model has {in_ch} input / {out_ch} output channels')
    if not (numpy.all(st[1] > 0) and numpy.all(st[3] > 0)):
        raise ValueError('stage-1 statistics: standard deviations must be positive')
    return st


class AcousticConverter(object):
    """Stage 1.  `gpu` is accepted for signature compatibility (converter/yukarin_converter.py:44);
    the engine always runs on the process's H100."""

    def __init__(self, config: Config, model_path: Path, gpu: int = None, f0_converter: F0Converter = None,
                 out_sampling_rate: int = None, engine: Optional[Engine] = None, feature_stats=None) -> None:
        self.config = config
        self.model_path = model_path
        self.gpu = gpu
        self.f0_converter = f0_converter
        self.out_sampling_rate = out_sampling_rate if out_sampling_rate is not None else config.dataset.acoustic_param.sampling_rate
        self.engine = engine or default_engine()
        params = load_npz(model_path)
        in_ch, out_ch, _ = upload_unet(self.engine, 1, params)
        self.in_mean, self.in_std, self.out_mean, self.out_std = load_stage1_stats(params, model_path, in_ch, out_ch, feature_stats)
        self.engine.stage1_set_stats(self.in_mean, self.in_std, self.out_mean, self.out_std)
        if f0_converter is not None:
            self.engine.f0_set_stats(*f0_converter.stats())

    # ---- the four calls VoiceChanger makes (voice_changer.py:27-38) ----
    def separate_effective(self, wave, feature: AcousticFeature, threshold):
        p = self.config.dataset.acoustic_param
        hop = p.sampling_rate * p.frame_period // 1000
        n = len(feature.f0)
        effective = self.engine.silence_mask(wave.wave, frame_length=p.fft_length, hop=hop, threshold_db=threshold, n_frames=n)
        return feature.indexing(effective), effective

    def convert(self, in_feature: AcousticFeature) -> AcousticFeature:
        mc = self.engine.stage1_convert(numpy.asarray(in_feature.mc, dtype=numpy.float32))
        voiced = numpy.asarray(in_feature.voiced, dtype=bool)
        f0_in = numpy.asarray(in_feature.f0, dtype=numpy.float32)
        if self.f0_converter is not None:
            self.engine.f0_set_stats(*self.f0_converter.stats())
            f0 = self.engine.f0_convert(f0_in.ravel(), voiced.ravel()).reshape(f0_in.shape)
        else:
            f0 = numpy.where(voiced, f0_in, 0).astype(numpy.float32)
        return AcousticFeature(f0=f0, mc=mc, ap=in_feature.ap, voiced=voiced)

    def combine_silent(self, effective: numpy.ndarray, feature: AcousticFeature) -> AcousticFeature:
        sizes = AcousticFeature.get_sizes(sampling_rate=self.out_sampling_rate, order=self.config.dataset.acoustic_param.order)
        out = AcousticFeature.silent(len(effective), sizes=sizes, keys=('mc', 'ap', 'f0', 'voiced'))
        if numpy.any(effective):
            out.mc[effective] = feature.mc
            out.ap[effective] = feature.ap
            out.f0[effective] = feature.f0
            out.voiced[effective] = feature.voiced
        return out

    def decode_spectrogram(self, feature: AcousticFeature) -> AcousticFeature:
        p = self.config.dataset.acoustic_param
        fftlen = cheaptrick_fft_size(self.out_sampling_rate)
        feature.sp = self.engine.mc2sp(numpy.asarray(feature.mc, dtype=numpy.float32), alpha=p.alpha, fftlen=fftlen)
        return feature


class SuperResolution(object):
    """Stage 2: (T, 513) float32 power spectrogram -> (T, 513) (voice_changer.py:41)."""

    def __init__(self, config: SRConfig, model_path: Path, gpu: int = None, engine: Optional[Engine] = None) -> None:
        self.config = config
        self.model_path = model_path
        self.gpu = gpu
        self.engine = engine or default_engine()
        upload_unet(self.engine, 2, load_npz(model_path))

    def convert(self, input: numpy.ndarray) -> numpy.ndarray:
        return self.engine.stage2_convert(numpy.asarray(input, dtype=numpy.float32))
