"""VoiceChanger: the per-window conversion of the hot path, with the constructor and method of
realtime_voice_conversion/yukarin_wrapper/voice_changer.py:8-42.

Two routes through the same kernels:
  * staged (default) -- silence gate, stage 1 (+ f0 map), scatter into the silent template, mc2sp, `+1e-16`, stage 2 as separate
    engine calls on host arrays, one call per step of voice_changer.py:27-41 (this is what the Stream classes use);
  * fused=True       -- the whole window in one upload / one download through ryk_convert_window.
`formant_ratio` warps the converted spectral envelope in the staged route (Engine.stage2_convert); the fused route has no warp."""
import numpy

from .feature import AcousticFeature, AcousticFeatureWrapper
from .models import AcousticConverter, SuperResolution

SP_FLOOR = 1e-16          # voice_changer.py:39: keeps log(sp) finite in stage 2 where mc2sp underflows


class VoiceChanger(object):
    def __init__(self, acoustic_converter: AcousticConverter, super_resolution: SuperResolution, threshold: float = 60,
                 output_sampling_rate: int = None, fused: bool = False, formant_ratio: float = 1.0) -> None:
        if fused and formant_ratio != 1.0:
            raise ValueError('the fused route has no formant warp: use the staged route (fused=False) for formant_ratio != 1')
        self.acoustic_converter = acoustic_converter
        self.super_resolution = super_resolution
        self.threshold = threshold
        self.output_sampling_rate = (output_sampling_rate if output_sampling_rate is not None
                                     else super_resolution.config.dataset.param.voice_param.sample_rate)
        self.fused = fused
        self.formant_ratio = float(formant_ratio)

    def convert_from_acoustic_feature(self, f_in: AcousticFeatureWrapper) -> AcousticFeature:
        return self._convert_fused(f_in) if self.fused else self._convert_staged(f_in)

    # ---- staged route ------------------------------------------------------------------------------------------
    def _stage1(self, f_in: AcousticFeatureWrapper) -> AcousticFeature:
        """Effective (non-silent) frames through the stage-1 net; silent frames keep the silent template."""
        ac = self.acoustic_converter
        effective_feature, mask = ac.separate_effective(wave=f_in.wave, feature=f_in, threshold=self.threshold)
        converted = ac.convert(effective_feature) if numpy.any(mask) else effective_feature      # nothing to convert in an all-silent window
        return ac.combine_silent(effective=mask, feature=converted)

    def _convert_staged(self, f_in: AcousticFeatureWrapper) -> AcousticFeature:
        f_out = self.acoustic_converter.decode_spectrogram(self._stage1(f_in))        # mel-cepstrum -> spectral envelope
        f_out.sp += SP_FLOOR
        f_out.sp = self.super_resolution.convert(f_out.sp.astype(numpy.float32), formant_ratio=self.formant_ratio)
        return f_out

    # ---- fused route -------------------------------------------------------------------------------------------
    def _convert_fused(self, f_in: AcousticFeatureWrapper) -> AcousticFeature:
        from .world_consts import cheaptrick_fft_size
        ac = self.acoustic_converter
        p = ac.config.dataset.acoustic_param
        out = ac.engine.convert_window(
            f_in.wave.wave, fs=p.sampling_rate, frame_length=p.fft_length, hop=p.sampling_rate * p.frame_period // 1000,
            threshold_db=self.threshold, f0=f_in.f0, ap=f_in.ap, mc=f_in.mc, voiced=f_in.voiced, order=p.order,
            alpha=p.alpha, fftlen=cheaptrick_fft_size(ac.out_sampling_rate))
        return AcousticFeature(f0=out['f0'][:, None], ap=out['ap'], sp=out['sp'], mc=out['mc'], voiced=out['voiced'][:, None])
