"""Window geometries of streaming sessions -- TEST INFRASTRUCTURE (no GPU).

A session derives its device layout from buffer_time, the encode / convert / decode extras and the frame period (csrc/session.cu
session_build), at 24 kHz: rate = 1000 / frame_period frames a second (200 at 5 ms; the period must divide 1000 ms) of hop =
24 * frame_period samples, n_feat = lrint(buffer_time * rate) frames per chunk, e_enc / e_conv / e_dec = lrint(extra * rate) frames, the
convert window Tw = n_feat + 2 e_conv, padded to Tp = Tw + 128 - Tw % 128 rows (always > Tw) for the U-Nets, Tp / 128 + 1 stage-1
buckets (at most 16), stage 2's kept rows [e_conv, e_conv + n_feat), the decode window Td = n_feat + 2 e_dec and the most samples one
step returns, (Td * hop // block + 4) whole synthesizer blocks.  Python's round() and C's lrint() both round halves to even.
"""
from dataclasses import dataclass
from typing import Tuple

FS = 24000
MAX_BUCKETS = 16               # bodies of a session's stage-1 SWITCH graph


@dataclass(frozen=True)
class Geometry:
    id: str
    buffer_time: float
    extra: Tuple[float, float, float]       # encode, convert, decode extra time (s)
    frame_period: float = 5.0               # ms

    @property
    def rate(self):
        return round(1000 / self.frame_period)

    @property
    def hop(self):
        return int(FS * self.frame_period / 1000)

    @property
    def n_feat(self):
        return round(self.buffer_time * self.rate)

    @property
    def n_wave(self):
        return round(self.buffer_time * FS)

    @property
    def e_wave(self):
        return round(self.extra[0] * FS)

    @property
    def e_enc(self):
        return round(self.extra[0] * self.rate)

    @property
    def e_conv(self):
        return round(self.extra[1] * self.rate)

    @property
    def e_dec(self):
        return round(self.extra[2] * self.rate)

    @property
    def Tw(self):
        return self.n_feat + 2 * self.e_conv

    @property
    def Tp(self):
        return self.Tw + 128 - self.Tw % 128

    @property
    def buckets(self):
        return self.Tp // 128 + 1

    @property
    def Td(self):
        return self.n_feat + 2 * self.e_dec

    def max_out(self, block=1024):
        """the most samples one step returns: the synthesizer's whole blocks of `block` samples"""
        return (self.Td * self.hop // block + 4) * block

    @property
    def keep(self):
        """stage 2's kept rows (begin, length): the chunk's frames of the convert window"""
        return self.e_conv, self.n_feat

    def session_config(self, threshold_db=60.0, block=1024):
        from realtime_yukarin_b200.engine import SessionConfig
        return SessionConfig(fs=FS, frame_period_ms=self.frame_period, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                             buffer_time=self.buffer_time, encode_extra_time=self.extra[0], convert_extra_time=self.extra[1],
                             decode_extra_time=self.extra[2], threshold_db=-1.0 if threshold_db is None else threshold_db,
                             vocoder_buffer_size=block)


GEOMETRIES = [
    Geometry('G1', 0.005, (0.0, 0.05, 0.0)),        # a one-frame chunk; 120-sample analysis windows
    Geometry('G2', 0.05, (0.025, 0.1, 0.025)),      # every extra non-zero, Td > n_feat
    Geometry('G3', 0.64, (0.0, 0.0, 0.0)),          # Tw % 128 == 0: a whole block of padding
    Geometry('G4', 0.635, (0.0, 0.0, 0.0)),         # one padding row
    Geometry('G5', 0.305, (0.05, 0.17, 0.02)),      # odd n_feat, Tw % 128 == 1
    Geometry('G6', 0.3, (0.0, 0.81, 0.0)),          # Tw % 128 == 0 at a larger size
    Geometry('G7', 1.0, (0.1, 2.0, 0.1)),           # large stage 2, extras on both sides
    Geometry('G8', 2.0, (0.0, 2.3, 0.0)),
    Geometry('G9', 0.305, (0.0, 4.645, 0.0)),       # 16 buckets: the largest accepted window
]
BY_ID = {g.id: g for g in GEOMETRIES}

# the shortest refused window: Tw 1920, Tp 2048, 17 buckets
TOO_LONG = Geometry('too-long', 0.3, (0.0, 4.65, 0.0))


def stage2_cases():
    """(Tp, keep_begin, keep_len, Tw) of every geometry"""
    return [(g.Tp, *g.keep, g.Tw) for g in GEOMETRIES]
