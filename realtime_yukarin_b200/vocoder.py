"""Vocoder / RealtimeVocoder: WORLD analysis and realtime synthesis on the H100.

Same constructor and methods as realtime_voice_conversion/yukarin_wrapper/vocoder.py:15-126; the
pyworld / world4py calls are replaced by libryk entry points (include/ryk.h).
"""
import numpy

from .config import VocodeMode
from .engine import Engine, default_engine
from .feature import AcousticFeature, AcousticFeatureWrapper, Wave
from .world_consts import cheaptrick_fft_size


class CrepeAcousticFeatureWrapper(AcousticFeatureWrapper):
    """CREPE f0 front-end (acoustic_feature_wrapper.py:65-80): crepe.predict + crepe.predict_voicing on the device (csrc/crepe.cu),
    the rest of the analysis (CheapTrick / D4C / sp2mc) on that f0.  Needs a weight file (realtime_yukarin_b200.crepe)."""

    @classmethod
    def extract_f0(cls, x, fs, frame_period, f0_floor, f0_ceil):
        from . import crepe
        return crepe.extract_f0(x, fs, frame_period)


class Vocoder(object):
    def __init__(self, acoustic_param, out_sampling_rate: int, extract_f0_mode: VocodeMode = VocodeMode.WORLD):
        self.acoustic_param = acoustic_param
        self.out_sampling_rate = out_sampling_rate
        self.extract_f0_mode = extract_f0_mode

    def encode(self, wave: Wave) -> AcousticFeatureWrapper:
        p = self.acoustic_param
        cls = AcousticFeatureWrapper if self.extract_f0_mode == VocodeMode.WORLD else CrepeAcousticFeatureWrapper
        return cls.extract(wave, frame_period=p.frame_period, f0_floor=p.f0_floor, f0_ceil=p.f0_ceil,
                           fft_length=p.fft_length, order=p.order, alpha=p.alpha, dtype=p.dtype)

    def decode(self, acoustic_feature: AcousticFeature) -> Wave:
        """Whole-utterance synthesis = pyworld.synthesize (vocoder.py:50-62): WORLD's offline Synthesis() on the device
        (ryk_world_synthesize); int(T * frame_period * fs / 1000) samples."""
        f = acoustic_feature
        out = default_engine().world_synthesize(numpy.asarray(f.f0, numpy.float64).ravel(), f.sp, f.ap, self.out_sampling_rate,
                                                self.acoustic_param.frame_period)
        return Wave(out, sampling_rate=self.out_sampling_rate)


class RealtimeVocoder(Vocoder):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._synthesizer = None
        self._engine: Engine = None
        self._buffer_size = None

    def create_synthesizer(self, buffer_size: int, number_of_pointers: int):
        assert self._synthesizer is None
        self._engine = default_engine()
        self._buffer_size = buffer_size
        self._synthesizer = self._engine.synth_create(
            self.out_sampling_rate, self.acoustic_param.frame_period,
            cheaptrick_fft_size(self.out_sampling_rate), buffer_size, number_of_pointers)

    def decode(self, acoustic_feature: AcousticFeature) -> Wave:
        assert self._synthesizer is not None
        f = acoustic_feature
        wave = self._engine.synth_decode(self._synthesizer, numpy.asarray(f.f0).ravel(), f.sp, f.ap)
        return Wave(wave=wave, sampling_rate=self.out_sampling_rate)

    def warm_up(self, time_length: float):
        y = numpy.zeros(int(time_length * self.out_sampling_rate))
        f = self.encode(Wave(wave=y, sampling_rate=self.out_sampling_rate))
        self.decode(f)
