"""Wave / AcousticFeature / AcousticFeatureWrapper: the value types that cross the Stream API.

Mirrors what the reference uses from `yukarin.wave.Wave` and `yukarin.acoustic_feature.AcousticFeature`
(un-vendored; semantics reconstructed from the call sites cited below) and re-creates
`AcousticFeatureWrapper` (realtime_voice_conversion/yukarin_wrapper/acoustic_feature_wrapper.py:8-62).

Pinned by the reference:
  * arrays are 2-D (frames, dim); f0 / voiced are (frames, 1)      tests/test_convert_stream.py:58-61
  * N frames <-> round(N * frame_period / 1000 * sr) samples         acoustic_feature_wrapper.py:43,57-58
  * wrapper equality = wave, sampling rate and f0                     acoustic_feature_wrapper.py:13-20
  * `obj.__dict__` round-trips through the constructor                acoustic_feature_wrapper.py:25,32,47,54,62
DECIDE (unpinned upstream): silent frames are f0=0, sp=0, ap=0, voiced=False and
mc = [SILENT_MC0, 0, ...] with SILENT_MC0 = ln(1e-8) so that mc2sp(silent) = 1e-16 (the magnitude of
the `+1e-16` guard at voice_changer.py:39); sp=0 silent frames are what makes the synthesizer emit
NaN that decode_stream.py:38 scrubs.
"""
from typing import Dict, Iterable, List, Optional, Sequence

import numpy

SILENT_MC0 = -18.420680743952367
_KEYS = ('f0', 'sp', 'ap', 'coded_ap', 'mc', 'voiced')


class Wave(object):
    def __init__(self, wave: numpy.ndarray, sampling_rate: int) -> None:
        self.wave = wave
        self.sampling_rate = sampling_rate

    def __len__(self):
        return len(self.wave)


def _is_missing(v) -> bool:
    return isinstance(v, float) and v != v


class AcousticFeature(object):
    all_keys = _KEYS

    def __init__(self, f0=numpy.nan, sp=numpy.nan, ap=numpy.nan, coded_ap=numpy.nan, mc=numpy.nan,
                 voiced=numpy.nan) -> None:
        self.f0 = f0
        self.sp = sp
        self.ap = ap
        self.coded_ap = coded_ap
        self.mc = mc
        self.voiced = voiced

    # aliases read by Vocoder.decode (vocoder.py:57-58)
    @property
    def spectrogram(self):
        return self.sp

    @property
    def aperiodicity(self):
        return self.ap

    # ---- shape bookkeeping -----------------------------------------------------------------
    @staticmethod
    def get_sizes(sampling_rate: int, order: int) -> Dict[str, int]:
        from .world_consts import cheaptrick_fft_size
        fft_size = cheaptrick_fft_size(sampling_rate)
        return dict(f0=1, sp=fft_size // 2 + 1, ap=fft_size // 2 + 1, coded_ap=max(1, min(15000, sampling_rate // 2 - 3000) // 3000),
                    mc=order + 1, voiced=1)

    @staticmethod
    def silent(length: int, sizes: Dict[str, int], keys: Iterable[str]) -> 'AcousticFeature':
        d = {}
        for k in keys:
            if k == 'voiced':
                d[k] = numpy.zeros((length, sizes[k]), dtype=bool)
            else:
                d[k] = numpy.zeros((length, sizes[k]), dtype=numpy.float32)
                if k == 'mc':
                    d[k][:, 0] = SILENT_MC0
        return AcousticFeature(**d)

    @staticmethod
    def concatenate(fs: Sequence['AcousticFeature'], keys: Optional[Iterable[str]] = None) -> 'AcousticFeature':
        keys = _KEYS if keys is None else keys
        # a key that is missing (NaN placeholder) on the inputs stays missing (the reference's own
        # tests concatenate / pick f0-only wrappers with the default 4-key list)
        return AcousticFeature(**{k: numpy.concatenate([getattr(f, k) for f in fs]) for k in keys
                                  if not any(_is_missing(getattr(f, k)) for f in fs)})

    def pick(self, first: int, last: int, keys: Optional[Iterable[str]] = None) -> 'AcousticFeature':
        keys = _KEYS if keys is None else keys
        return AcousticFeature(**{k: getattr(self, k)[first:last] for k in keys if not _is_missing(getattr(self, k))})

    def indexing(self, index: numpy.ndarray) -> 'AcousticFeature':
        return AcousticFeature(**{k: v[index] for k, v in self._present()})

    def _present(self):
        return [(k, getattr(self, k)) for k in _KEYS if not _is_missing(getattr(self, k))]

    # ---- dtype helpers ---------------------------------------------------------------------
    def astype(self, dtype) -> 'AcousticFeature':
        return AcousticFeature(**{k: (v.astype(dtype) if hasattr(v, 'astype') else v)
                                  for k, v in self.__dict__.items() if k in _KEYS})

    def astype_only_float(self, dtype) -> 'AcousticFeature':
        d = {}
        for k in _KEYS:
            v = getattr(self, k)
            if hasattr(v, 'astype') and k != 'voiced':
                v = v.astype(dtype)
            d[k] = v
        return AcousticFeature(**d)

    def validate(self) -> None:
        n = None
        for k, v in self._present():
            assert v.ndim == 2, k
            n = len(v) if n is None else n
            assert len(v) == n, k

    # ---- WORLD analysis (SURVEY a6; vocoder.py:28-37 -> acoustic_feature_wrapper.py:28-33) ----
    @classmethod
    def extract_f0(cls, x: numpy.ndarray, fs: int, frame_period: int, f0_floor: float, f0_ceil: float):
        """DIO + StoneMask on the H100 (hook kept so that subclasses can swap the f0 front-end,
        as acoustic_feature_wrapper.py:66-80 does)."""
        from .engine import default_engine
        return default_engine().world_f0(x, fs, frame_period, f0_floor, f0_ceil)

    @classmethod
    def extract(cls, wave: Wave, frame_period, f0_floor, f0_ceil, fft_length, order, alpha, dtype) -> 'AcousticFeature':
        from .engine import default_engine
        x = numpy.asarray(wave.wave)
        f0_in = None
        if cls.extract_f0.__func__ is not AcousticFeature.extract_f0.__func__:
            f0_in, _ = cls.extract_f0(x.astype(numpy.float64), wave.sampling_rate, frame_period, f0_floor, f0_ceil)
        out = default_engine().world_analyze(
            x, fs=wave.sampling_rate, frame_period=frame_period, f0_floor=f0_floor, f0_ceil=f0_ceil,
            fft_length=fft_length, order=order, alpha=alpha, f0=f0_in)
        f = AcousticFeature(f0=out['f0'][:, None], sp=out['sp'], ap=out['ap'], mc=out['mc'],
                            voiced=out['voiced'][:, None])
        return f.astype_only_float(dtype)


class AcousticFeatureWrapper(AcousticFeature):
    """An AcousticFeature that drags the sample-aligned input waveform along (the silence gate of
    stage 1 needs it: voice_changer.py:25-31)."""

    def __init__(self, wave: Wave, *args, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.wave = wave

    def __eq__(self, other):
        if not isinstance(other, AcousticFeatureWrapper):
            return NotImplemented
        return bool(
            numpy.all(other.wave.wave == self.wave.wave)
            and other.wave.sampling_rate == self.wave.sampling_rate
            and numpy.all(other.f0 == self.f0)
        )

    __hash__ = None

    def _feature_kwargs(self, feature: AcousticFeature) -> dict:
        return {k: getattr(feature, k) for k in _KEYS}

    def astype_only_float_wrapper(self, dtype) -> 'AcousticFeatureWrapper':
        w = Wave(wave=self.wave.wave.astype(dtype), sampling_rate=self.wave.sampling_rate)
        return AcousticFeatureWrapper(wave=w, **self._feature_kwargs(self.astype_only_float(dtype)))

    @classmethod
    def extract(cls, wave: Wave, *args, **kwargs) -> 'AcousticFeatureWrapper':
        base = super().extract(wave, *args, **kwargs)
        return cls(wave=wave, **{k: getattr(base, k) for k in _KEYS})

    @staticmethod
    def silent_wrapper(length: int, sizes: Dict[str, int], keys: Iterable[str], frame_period: float,
                       sampling_rate: int, wave_dtype) -> 'AcousticFeatureWrapper':
        n_samples = round(length * frame_period / 1000 * sampling_rate)
        feature = AcousticFeature.silent(length, sizes=sizes, keys=keys)
        return AcousticFeatureWrapper(
            wave=Wave(wave=numpy.zeros(shape=n_samples, dtype=wave_dtype), sampling_rate=sampling_rate),
            **{k: getattr(feature, k) for k in _KEYS})

    @staticmethod
    def concatenate_wrapper(fs: List['AcousticFeatureWrapper'], keys: Iterable[str]) -> 'AcousticFeatureWrapper':
        feature = AcousticFeature.concatenate(fs, keys=keys)
        wave = numpy.concatenate([f.wave.wave for f in fs])
        return AcousticFeatureWrapper(wave=Wave(wave=wave, sampling_rate=fs[0].wave.sampling_rate),
                                      **{k: getattr(feature, k) for k in _KEYS})

    def pick_wrapper(self, first: int, last: int, keys: Iterable[str], frame_period: float) -> 'AcousticFeatureWrapper':
        sr = self.wave.sampling_rate
        lo = round(first * frame_period / 1000 * sr)
        hi = round(last * frame_period / 1000 * sr)
        feature = self.pick(first, last, keys=keys)
        return AcousticFeatureWrapper(wave=Wave(wave=self.wave.wave[lo:hi], sampling_rate=sr),
                                      **{k: getattr(feature, k) for k in _KEYS})
