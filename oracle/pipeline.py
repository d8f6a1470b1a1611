"""CPU restatement of the whole per-chunk hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

encode  : yukarin.AcousticFeature.extract                      (vocoder.py:26-48 -> acoustic_feature_wrapper.py:28-33; SURVEY A.1)
convert : VoiceChanger.convert_from_acoustic_feature           (voice_changer.py:24-42; SURVEY A.6, A.7)
decode  : RealtimeVocoder.decode + NaN scrub                   (vocoder.py:89-120, decode_stream.py:38; SURVEY A.8)
stream  : the EncodeStream/ConvertStream/DecodeStream + StreamWrapper chain as the workers drive it
          (worker/encode_worker.py:31-40 etc.), restated through the closed-form window identity of
          SURVEY A.9a instead of the segment store, so that it is independent of the product's stream.py.
PARITY UNPINNED (see oracle/world_oracle.c).  DECIDE points mirrored from DESIGN.md:
  f0 = DIO + StoneMask; frames trimmed to len(x) // hop; silence gate = librosa reflect-padded frame MSE,
  ref = max over the window, fp64; silent template mc0 = ln(1e-8); F0 conversion in fp64 -> fp32.
"""
from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import numpy as np

from . import nets
from . import world as W

SILENT_MC0 = -18.420680743952367


@dataclass
class PathConfig:
    fs: int = 24000
    frame_period: float = 5.0
    f0_floor: float = 71.0
    f0_ceil: float = 800.0
    fft_length: int = 1024
    order: int = 8
    alpha: float = 0.466
    threshold_db: Optional[float] = 60.0
    vocoder_buffer_size: int = 1024
    f0_method: str = 'dio'        # 'dio' | 'harvest' (yukarin's f0_estimating_method; both are followed by StoneMask)

    @property
    def hop(self) -> int:
        return int(self.fs * self.frame_period / 1000)


def extract_features(wave: np.ndarray, cfg: PathConfig) -> Dict[str, np.ndarray]:
    x = np.asarray(wave).astype(np.float64)
    n_out = len(x) // cfg.hop
    nb = cfg.fft_length // 2 + 1
    if n_out == 0:
        return dict(f0=np.zeros((0, 1), np.float32), sp=np.zeros((0, nb), np.float32), ap=np.zeros((0, nb), np.float32),
                    mc=np.zeros((0, cfg.order + 1), np.float32), voiced=np.zeros((0, 1), bool))
    if cfg.f0_method == 'harvest':
        f0, t = W.harvest(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil)
    else:
        f0, t = W.dio(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil)
    f0 = W.stonemask(x, cfg.fs, t, f0)
    sp = W.cheaptrick(x, cfg.fs, t, f0, cfg.fft_length)
    ap = W.d4c(x, cfg.fs, t, f0, cfg.fft_length)
    mc = W.sp2mc(sp, cfg.order, cfg.alpha)
    voiced = ~(f0 == 0)
    return dict(f0=f0[:n_out, None].astype(np.float32), sp=sp[:n_out].astype(np.float32), ap=ap[:n_out].astype(np.float32),
                mc=mc[:n_out].astype(np.float32), voiced=voiced[:n_out, None])


def effective_mask(wave: np.ndarray, n_frames: int, cfg: PathConfig, threshold_db) -> np.ndarray:
    if threshold_db is None:
        return np.ones(n_frames, dtype=bool)
    mse = W.frame_mse(wave, cfg.fft_length, cfg.hop, n_frames)
    if n_frames == 0:
        return np.zeros(0, dtype=bool)
    ref = 10.0 * np.log10(max(1e-10, float(mse.max())))
    db = 10.0 * np.log10(np.maximum(1e-10, mse)) - ref
    return db > -threshold_db


def f0_convert(f0: np.ndarray, voiced: np.ndarray, stats) -> np.ndarray:
    mu_i, sd_i, mu_t, sd_t = stats
    f = np.asarray(f0, dtype=np.float32).ravel()
    v = np.asarray(voiced, dtype=bool).ravel()
    out = np.zeros_like(f)
    out[v] = np.exp((np.log(f[v].astype(np.float64)) - mu_i) / sd_i * sd_t + mu_t).astype(np.float32)
    return out


def convert_window(wave: np.ndarray, feat: Dict[str, np.ndarray], cfg: PathConfig, stage1, stage2, f0_stats,
                   backend: str = 'numpy', threshold_db='cfg') -> Dict[str, np.ndarray]:
    """voice_changer.py:24-42 on one window. feat: f0 (T,1), ap (T,nb), mc (T,C), voiced (T,1)."""
    thr = cfg.threshold_db if threshold_db == 'cfg' else threshold_db
    T = len(feat['f0'])
    nb = cfg.fft_length // 2 + 1
    C = cfg.order + 1
    eff = effective_mask(wave, T, cfg, thr)
    mc = np.zeros((T, C), np.float32)
    mc[:, 0] = SILENT_MC0
    ap = np.zeros((T, nb), np.float32)
    f0 = np.zeros((T, 1), np.float32)
    voiced = np.zeros((T, 1), bool)
    if eff.any():
        mc[eff] = nets.stage1_convert(feat['mc'][eff], stage1, backend)
        v = feat['voiced'][eff]
        f0[eff] = f0_convert(feat['f0'][eff], v, f0_stats)[:, None]
        ap[eff] = feat['ap'][eff]
        voiced[eff] = v
    sp = W.mc2sp(mc.astype(np.float32), cfg.alpha, cfg.fft_length)
    sp += 1e-16
    sp_mid = sp.astype(np.float32)
    sp_out = nets.stage2_convert(sp_mid, stage2, backend)
    return dict(f0=f0, ap=ap, sp=sp_out, voiced=voiced, mc=mc, sp_mid=sp_mid, effective=eff)


class StreamOracle:
    """One audio stream pushed chunk by chunk through encode -> convert -> decode with the
    reference's overlap ("extra_time") semantics; index math per SURVEY A.9a:
    stage window element i of step k == input item k*n - 2e + i (silent / zero where negative)."""

    def __init__(self, cfg: PathConfig, stage1, stage2, f0_stats, buffer_time=0.3, extra=(0.0, 0.5, 0.0), backend='numpy'):
        self.cfg, self.stage1, self.stage2, self.f0_stats, self.backend = cfg, stage1, stage2, f0_stats, backend
        self.buffer_time = buffer_time
        self.extra = extra
        self.rate = round(1000 / cfg.frame_period)
        self.n_wave = round(buffer_time * cfg.fs)
        self.n_feat = round(buffer_time * self.rate)
        self.e_wave = round(extra[0] * cfg.fs)
        self.e_conv = round(extra[1] * self.rate)
        self.e_dec = round(extra[2] * self.rate)
        self.k = 0
        self.wave_base = self.enc_base = self.conv_base = 0       # rows already dropped from the front of the histories (long soak runs)
        self.wave_hist = np.zeros(0, np.float32)
        nb = cfg.fft_length // 2 + 1
        self.enc_hist = dict(f0=np.zeros((0, 1), np.float32), ap=np.zeros((0, nb), np.float32),
                             mc=np.zeros((0, cfg.order + 1), np.float32), voiced=np.zeros((0, 1), bool), wave=np.zeros(0, np.float32))
        self.conv_hist = dict(f0=np.zeros((0, 1), np.float32), ap=np.zeros((0, nb), np.float32), sp=np.zeros((0, nb), np.float32))
        self.synth = W.RealtimeSynthesizer(cfg.fs, cfg.frame_period, W.cheaptrick_fft_size(cfg.fs), cfg.vocoder_buffer_size)

    @staticmethod
    def _window(arr, first, length, fill):
        """rows [first, first+length) of arr; rows outside [0, len) take `fill` (one row)."""
        out = np.empty((length,) + arr.shape[1:], dtype=arr.dtype)
        out[...] = fill
        lo, hi = max(first, 0), min(first + length, len(arr))
        if hi > lo:
            out[lo - first:hi - first] = arr[lo:hi]
        return out

    def _extract(self, win: np.ndarray) -> Dict[str, np.ndarray]:
        """the encode stage on one encode window; a subclass may put another implementation of the same stage here"""
        return extract_features(win, self.cfg)

    def _convert(self, wave: np.ndarray, feat: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
        """the convert stage on one convert window (wave: its Tw * hop samples); a subclass may put another implementation here"""
        return convert_window(wave, feat, self.cfg, self.stage1, self.stage2, self.f0_stats, self.backend)

    def push(self, chunk: np.ndarray):
        cfg, k = self.cfg, self.k
        hop = cfg.hop
        nb = cfg.fft_length // 2 + 1
        assert len(chunk) == self.n_wave
        # ---- encode ----
        self.wave_hist = np.concatenate([self.wave_hist, np.asarray(chunk, np.float32)])
        win = self._window(self.wave_hist, k * self.n_wave - 2 * self.e_wave - self.wave_base, self.n_wave + 2 * self.e_wave, 0.0)
        f = self._extract(win)
        pad = round(self.extra[0] * self.rate)
        aligned = win
        if pad > 0:
            f = {kk: v[pad:-pad] for kk, v in f.items()}
            aligned = win[round(pad * cfg.frame_period / 1000 * cfg.fs):round(-pad * cfg.frame_period / 1000 * cfg.fs)]
        for kk in ('f0', 'ap', 'mc', 'voiced'):
            self.enc_hist[kk] = np.concatenate([self.enc_hist[kk], f[kk]])
        self.enc_hist['wave'] = np.concatenate([self.enc_hist['wave'], aligned])
        # ---- convert ----
        Tw = self.n_feat + 2 * self.e_conv
        first = k * self.n_feat - 2 * self.e_conv - self.enc_base
        silent_mc = np.zeros((1, cfg.order + 1), np.float32)
        silent_mc[0, 0] = SILENT_MC0
        wfeat = dict(f0=self._window(self.enc_hist['f0'], first, Tw, 0.0), ap=self._window(self.enc_hist['ap'], first, Tw, 0.0),
                     mc=self._window(self.enc_hist['mc'], first, Tw, silent_mc), voiced=self._window(self.enc_hist['voiced'], first, Tw, False))
        wwave = self._window(self.enc_hist['wave'], first * hop, Tw * hop, 0.0)
        conv = self._convert(wwave, wfeat)
        if self.e_conv > 0:
            conv = {kk: v[self.e_conv:-self.e_conv] for kk, v in conv.items() if kk in ('f0', 'ap', 'sp')}
        for kk in ('f0', 'ap', 'sp'):
            self.conv_hist[kk] = np.concatenate([self.conv_hist[kk], conv[kk]])
        # ---- decode ----
        Td = self.n_feat + 2 * self.e_dec
        firstd = k * self.n_feat - 2 * self.e_dec - self.conv_base
        df0 = self._window(self.conv_hist['f0'], firstd, Td, 0.0)
        dsp = self._window(self.conv_hist['sp'], firstd, Td, 0.0)
        dap = self._window(self.conv_hist['ap'], firstd, Td, 0.0)
        y = self.synth.decode(df0.ravel().astype(np.float64), dsp, dap)
        y = np.array(y)
        y[np.isnan(y)] = 0
        self.k += 1
        self.last = dict(encoded=f, converted=conv)
        # drop history no window can reach any more (rows before the next step's first row); negative window indices stay "silent"
        keep_w = (self.k * self.n_wave - 2 * self.e_wave) - self.wave_base
        if keep_w > 8 * (self.n_wave + 2 * self.e_wave):
            self.wave_hist = self.wave_hist[keep_w:]; self.wave_base += keep_w
        keep_e = (self.k * self.n_feat - 2 * self.e_conv) - self.enc_base
        if keep_e > 8 * (self.n_feat + 2 * self.e_conv):
            for kk in ('f0', 'ap', 'mc', 'voiced'):
                self.enc_hist[kk] = self.enc_hist[kk][keep_e:]
            self.enc_hist['wave'] = self.enc_hist['wave'][keep_e * hop:]
            self.enc_base += keep_e
        keep_c = (self.k * self.n_feat - 2 * self.e_dec) - self.conv_base
        if keep_c > 8 * (self.n_feat + 2 * self.e_dec):
            for kk in ('f0', 'ap', 'sp'):
                self.conv_hist[kk] = self.conv_hist[kk][keep_c:]
            self.conv_base += keep_c
        return y


class OutputReblockOracle:
    """decode_worker.py:38-59 restated: `wave_fragment` accumulation, one out_audio_chunk per step, and the output silence
    gate power_to_db(abs(stft(chunk)) ** 2).mean() < -threshold (oracle/world.py: stft_power_db_mean)."""

    def __init__(self, out_audio_chunk: int, output_silent_threshold: float):
        self.chunk = int(out_audio_chunk)
        self.threshold = float(output_silent_threshold)
        self.fragment = np.empty(0)
        self.last_power = None

    def push(self, wave: np.ndarray) -> Tuple[int, Optional[np.ndarray]]:
        """-> (status, chunk): 0 = not enough samples yet, 1 = chunk, 2 = silent chunk (the reference forwards None)."""
        self.fragment = np.concatenate([self.fragment, np.asarray(wave, np.float64)])
        if len(self.fragment) < self.chunk:
            self.last_power = None
            return 0, None
        wave, self.fragment = self.fragment[:self.chunk], self.fragment[self.chunk:]
        self.last_power = W.stft_power_db_mean(wave)
        if self.last_power < -self.threshold:
            return 2, None
        return 1, wave
