"""realtime_yukarin_b200: the per-chunk hot path of realtime-yukarin (encode -> stage 1 -> stage 2 -> vocode)
on NVIDIA H100 (sm_90a), behind the reference's Stream / SegmentMethod plugin API and its
Vocoder / VoiceChanger / AcousticConverter / SuperResolution call surface.  See DESIGN.md.

`import realtime_yukarin_b200.dropin; realtime_yukarin_b200.dropin.install()` registers
`realtime_voice_conversion`, `yukarin` and `become_yukarin` import aliases so that the reference's
check.py-style drivers and unit tests run unchanged against this package.
"""
from .config import Config, VocodeMode  # noqa: F401
from .feature import AcousticFeature, AcousticFeatureWrapper, Wave  # noqa: F401
from .params import AcousticParam, Param  # noqa: F401
from .segment import (BaseSegmentMethod, FeatureSegmentMethod, FeatureWrapperSegmentMethod, Segment,  # noqa: F401
                      WaveSegmentMethod)
from .stream import BaseStream, ConvertStream, DecodeStream, EncodeStream, StreamWrapper  # noqa: F401
from .wave_io import load_wave, save_wave  # noqa: F401
from .worker import Item, OutputReblocker, RealtimePipeline  # noqa: F401

__version__ = '0.1.0'
