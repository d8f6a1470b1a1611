"""The reference's worker pipeline re-cast for one GPU (SURVEY 8(f) ranks 1 and 2).

The reference runs encode / convert / decode in three OS processes connected by queues of
`Item{item, index}` (run.py:58-93, worker/encode_worker.py, convert_worker.py, decode_worker.py); the
audio loop pushes one input chunk per iteration and pops whatever output is ready, re-ordering by
index (run.py:152-199).  Here the three stages are CUDA streams of one device-resident session
(csrc/session.cu), so the "queues" are tickets of chunks in flight:

  Item                              worker/utility.py:6-14
  OutputReblocker                   decode_worker.py:38-59 (wave_fragment re-blocking + output silence gate), fragment
                                    and STFT gate on the device (ryk_reblock_*)
  RealtimePipeline.put / get_nowait queue_input_wave.put / queue_output_wave.get_nowait (run.py:165, 176-182)
  RealtimePipeline.process          one iteration of the audio loop body (run.py:160-199) without PyAudio

Start offsets: the reference starts every worker at `start_time = extra_time` (encode_worker.py:31); the session
pre-fills its windows with silence for exactly those offsets.
"""
import json
import logging
import math
import os
import time
from collections import deque
from typing import Any, Deque, List, Optional, Tuple

import numpy

from .config import Config, VocodeMode
from .drift import DriftController
from .engine import (AGC_GATE_DB, AGC_MAX_GAIN_DB, AGC_TARGET_DB, DRIFT_MAX_PPM, LIMITER_CEILING_DB, LIMITER_HOLD_MS, LIMITER_LOOKAHEAD_MS,
                     PITCH_A4_HZ, PITCH_RETUNE_MS, Engine, SessionConfig, default_engine, pitch_key, pitch_scale)
from .wave_io import DRIFT_HALF_WIDTH


class Item(object):
    """worker/utility.py:6-14"""

    def __init__(self, item: Any, index: int):
        self.item = item
        self.index = index


def init_logger(logger=None, filename: Optional[str] = None):
    """worker/utility.py:16-29: level from $LOG_LEVEL (default WARNING), '%(levelname)s\\t%(name)s\\t%(asctime)s\\t%(message)s' on the
    console and -- when `filename` is given (the reference always writes ./log.txt) -- to that file."""
    if logger is None:
        logger = logging.getLogger()
    fmt = logging.Formatter('%(levelname)s\t%(name)s\t%(asctime)s\t%(message)s')
    logger.setLevel(os.getenv('LOG_LEVEL', 'WARNING'))
    if filename:
        handler = logging.FileHandler(filename)
        handler.setFormatter(fmt)
        logger.addHandler(handler)
    handler = logging.StreamHandler()
    handler.setFormatter(fmt)
    logger.addHandler(handler)
    return logger


class OutputReblocker(object):
    """decode_worker.py:38-59: queue synthesizer blocks, cut one `out_audio_chunk` per step, drop silent chunks."""

    def __init__(self, out_audio_chunk: int, output_silent_threshold: float, max_in: Optional[int] = None,
                 engine: Optional[Engine] = None):
        self.engine = engine or default_engine()
        self.out_audio_chunk = int(out_audio_chunk)
        self.output_silent_threshold = float(output_silent_threshold)
        self.max_in = int(max_in) if max_in else 2 * self.out_audio_chunk + 8192
        self._rid = self.engine.reblock_create(self.out_audio_chunk, self.max_in, self.output_silent_threshold)
        self.last_power = None
        self.last_status = 0

    def push(self, wave) -> Optional[numpy.ndarray]:
        """`wave` = what DecodeStream produced this step; returns the chunk to play or None (not enough samples / silent)."""
        status, chunk, power = self.engine.reblock_push(self._rid, numpy.asarray(wave, dtype=numpy.float64))
        self.last_status, self.last_power = status, power
        return chunk

    def close(self):
        if self._rid is not None:
            self.engine.reblock_destroy(self._rid)
            self._rid = None


def model_frame_period(acoustic_param) -> float:
    """The stream's frame period in ms: the stage-1 model's acoustic_param.frame_period (5 without one), as the reference builds its
    vocoder and its three streams from it (run.py:41, encode_stream.py:21, convert_stream.py:19, decode_stream.py:17).  Config's
    frame_period is read and not used, in the reference too."""
    return float(getattr(acoustic_param, 'frame_period', 5))


def _check_limiter(ceiling_db: float, output_scale: float, lookahead_ms: float, hold_ms: float) -> None:
    """the limiter's settings as Engine.session_limiter / session_set_limiter accept them, checked before a session exists"""
    lo, hi = LIMITER_CEILING_DB
    if not lo <= ceiling_db <= hi:
        raise ValueError(f'the limiter ceiling must be within [{lo}, {hi}] dB')
    if not (math.isfinite(output_scale) and output_scale > 0):
        raise ValueError('the limiter needs a finite, positive output_scale')
    lo, hi = LIMITER_LOOKAHEAD_MS
    if not lo <= lookahead_ms <= hi:
        raise ValueError(f'the limiter look-ahead must be within [{lo}, {hi}] ms')
    lo, hi = LIMITER_HOLD_MS
    if not lo <= hold_ms <= hi:
        raise ValueError(f'the limiter hold must be within [{lo}, {hi}] ms')


def _check_agc(target_db: float, max_gain_db: float, gate_db: float) -> None:
    """the AGC's settings as Engine.session_agc accepts them, checked before a session exists"""
    for name, v, (lo, hi) in (('target', target_db, AGC_TARGET_DB), ('maximum gain', max_gain_db, AGC_MAX_GAIN_DB),
                              ('gate', gate_db, AGC_GATE_DB)):
        if not lo <= v <= hi:
            raise ValueError(f'the AGC {name} must be within [{lo}, {hi}] dB')


PITCH_CORRECT_KEYS = ('key', 'scale', 'a4_hz', 'retune_ms', 'amount')


def pitch_settings(settings: dict) -> dict:
    """pitch correction settings as Engine.session_set_pitch_correct accepts them (key as 0-11, scale as a mask), checked before a
    session exists"""
    unknown = set(settings) - set(PITCH_CORRECT_KEYS)
    if unknown:
        raise ValueError(f'unknown pitch correction settings {sorted(unknown)}: use {", ".join(PITCH_CORRECT_KEYS)}')
    out = dict(key=0, scale='chromatic', a4_hz=440.0, retune_ms=50.0, amount=1.0)
    out.update(settings)
    out['key'], out['scale'] = pitch_key(out['key']), pitch_scale(out['scale'])
    if not 0 <= out['key'] <= 11:
        raise ValueError('the pitch correction key must be a pitch class within [0, 11]')
    if not 1 <= out['scale'] <= 0xfff:
        raise ValueError('the pitch correction scale must be a nonzero 12-bit mask')
    for name, (lo, hi) in (('a4_hz', PITCH_A4_HZ), ('retune_ms', PITCH_RETUNE_MS), ('amount', (0.0, 1.0))):
        out[name] = float(out[name])
        if not lo <= out[name] <= hi:
            raise ValueError(f'the pitch correction {name} must be within [{lo:g}, {hi:g}]')
    return out


def _check_drift(drift, max_ppm: float) -> None:
    """the drift stage's settings as Engine.drift_create / drift_set accept them, checked before a session exists"""
    if not (math.isfinite(max_ppm) and 0 < max_ppm <= DRIFT_MAX_PPM):
        raise ValueError(f'drift_max_ppm must be within (0, {DRIFT_MAX_PPM:g}]')
    if isinstance(drift, str):
        if drift != 'auto':
            raise ValueError("drift must be None, 'auto' or a trim in ppm")
    elif not (math.isfinite(float(drift)) and abs(float(drift)) <= max_ppm):
        raise ValueError('the drift trim must be finite and within +-drift_max_ppm')


class RealtimePipeline(object):
    """encode_worker | convert_worker | decode_worker of one audio stream as one device-resident session.

    The models must already be loaded into `engine` (YukarinConverter.make_yukarin_converter does that for voice 0,
    models.load_voice for any voice); the session converts into `voice`.  `depth` chunks may be in flight (the reference's queues
    are unbounded; the session keeps up to 5 steps in flight).

    `measure_f0=True` keeps running statistics of the speaker's log-f0 on the device (`measured_f0`); `follow_f0=N` (implies
    measuring) also makes them the input side of the session's f0 map once N voiced frames are counted.  `set_f0_map` changes the
    map between chunks.  `formant` (semitones, [-12, 12]) warps the converted spectral envelope from the first chunk on; `set_formant`
    changes it between chunks.  `denoise=DB` filters the input's noise ahead of the analysis (at most DB of attenuation, 0-40), with
    `noise_profile` (257 values, as `noise_profile()` returns them) or a profile learned from the first `learn_noise` seconds of input;
    `set_denoise` changes the reduction between chunks.  `echo_cancel=True` removes the echo of the played output from the input ahead of
    the analysis (and of the noise filter), for a voice played through speakers: `echo_taps` frames of 128 model samples (1-64) after a
    bulk delay of `echo_delay_ms` cover the echo path, and `echo_suppression` dB (0-40) of residual-echo suppression follows;
    `set_echo_suppression` changes it between chunks and `echo_stats` reads how much echo the last chunk lost.  The far end is what
    `process` returned: mic chunk i is paired with the next n_in samples of the played stream, which starts with one input chunk of
    zeros (chunk i with the output of chunk i - 1 when the chunk sizes are equal; silence where the output ran short).  It needs
    input_rate == output_rate.  `limiter=CEILING_DB` (-24 to 0) keeps the played samples (the session's times output_scale) under
    that ceiling with a look-ahead peak limiter on the device: `limiter_lookahead_ms` (0.5-10) of look-ahead, which the output delay
    grows by, and `limiter_hold_ms` (0-500) of hold; `set_limiter` changes the ceiling between chunks and `limiter_stats` reads how
    much the last chunk was limited.  With echo_cancel the far end is then the limited played stream.  `agc=TARGET_DB` (-40 to -6)
    brings the speaker's level (mean square, dB of full scale) to that target ahead of the analysis with an automatic gain control on the
    device, after the echo canceller and the noise filter: at most `agc_max_gain_db` (0-30) of gain either way, counting only the
    256-sample blocks louder than `agc_gate_db` (-80 to -20).  It follows `input_scale`: the host still multiplies each chunk by it
    first, so the gate applies to the scaled signal.  `set_agc` changes the settings between chunks and `agc_stats` reads the level
    and gain.  `drift` compensates the clock difference of two sound cards (DESIGN.md §4l): a drift stage on the device resamples the
    played stream so that it runs (1 + ppm 1e-6) times as long, with `drift=PPM` a fixed trim and `drift='auto'` a trim that
    `update_drift` derives from the output card's backlog; |ppm| <= `drift_max_ppm` (at most 2000).  `process` then returns the stage's
    output for the chunk it would have played: float32, one or two samples more or less than out_audio_chunk, 16 samples later.  The
    echo canceller's far end stays the chunk before the stage: the microphone hears the played sound in the input card's clock, which
    the nominal-rate stream is in.  `set_drift` fixes the trim, `drift_stats` reads it with the stage's totals.  `pitch_correct=dict(
    key=, scale=, a4_hz=, retune_ms=, amount=)` pulls each converted note toward the nearest note of a scale on the device (DESIGN.md
    §4m): key 0-11 or a note name ('C' when missing), scale a 12-bit mask or 'chromatic' (default) / 'major' / 'minor', a4_hz 400-480
    (440), retune_ms 0-1000 (50; 0 is a hard snap) and amount 0-1 (1); no delay.  `set_pitch_correct` changes the settings between
    chunks and `pitch_stats` reads how much the last chunk was corrected."""

    _drift: Optional[int] = None                        # the drift stage's id on the engine (None: no drift stage)
    _drift_ctl: Optional[DriftController] = None        # its controller in 'auto' mode

    def __init__(self, config: Config, acoustic_param=None, engine: Optional[Engine] = None, depth: int = 3, voice: int = 0,
                 measure_f0: bool = False, follow_f0: Optional[int] = None, formant: float = 0.0, denoise: Optional[float] = None,
                 noise_profile=None, learn_noise: Optional[float] = None, echo_cancel: bool = False, echo_taps: int = 32,
                 echo_delay_ms: float = 0.0, echo_suppression: float = 0.0, limiter: Optional[float] = None,
                 limiter_lookahead_ms: float = 5.0, limiter_hold_ms: float = 50.0, agc: Optional[float] = None,
                 agc_max_gain_db: float = 20.0, agc_gate_db: float = -50.0, drift=None, drift_max_ppm: float = 500.0,
                 pitch_correct: Optional[dict] = None):
        if pitch_correct is not None:
            pitch_correct = pitch_settings(pitch_correct)
        if drift is not None:
            _check_drift(drift, float(drift_max_ppm))
        if agc is not None:
            _check_agc(float(agc), float(agc_max_gain_db), float(agc_gate_db))
        if limiter is not None:
            _check_limiter(float(limiter), float(config.output_scale), float(limiter_lookahead_ms), float(limiter_hold_ms))
        if echo_cancel and int(config.input_rate) != int(config.output_rate):
            raise ValueError('echo_cancel needs input_rate == output_rate: the played stream is the far end of the input')
        self.config = config
        self.engine = engine or default_engine()
        p = acoustic_param
        # analysis, the U-Nets and synthesis run at the models' rate and frame period; the sound card's rates are the session's device
        # rates
        fs = int(getattr(p, 'sampling_rate', 24000))
        frame_period = model_frame_period(p)
        cfg = SessionConfig(
            fs=fs, frame_period_ms=frame_period,
            f0_floor=float(getattr(p, 'f0_floor', 71.0)), f0_ceil=float(getattr(p, 'f0_ceil', 800.0)),
            fft_length=int(getattr(p, 'fft_length', 1024)), order=int(getattr(p, 'order', 8)), alpha=float(getattr(p, 'alpha', 0.466)),
            buffer_time=float(config.buffer_time), encode_extra_time=float(config.encode_extra_time),
            convert_extra_time=float(config.convert_extra_time), decode_extra_time=float(config.decode_extra_time),
            threshold_db=float(config.input_silent_threshold), vocoder_buffer_size=int(config.vocoder_buffer_size))
        self.depth = max(1, min(int(depth), 5))
        # per-item stage timing at DEBUG, as the reference's workers log it (encode_worker.py:34,44, convert_worker.py:47,59,
        # decode_worker.py:42,66: `logger.debug(f'{item.index}: {time.time() - start}')` on loggers 'encode' / 'convert' / 'decode').
        # Here the stages are CUDA streams, so the figures are device times between CUDA events (ryk_session_stage_times).
        self._loggers = {k: logging.getLogger(k) for k in ('encode', 'convert', 'decode')}
        self._timing = any(lg.isEnabledFor(logging.DEBUG) for lg in self._loggers.values())
        # extract_f0_mode: crepe (run.py:40-44 hands it to the encode worker's Vocoder) analyses each encode window with CREPE
        # instead of DIO.  The session takes the engine's f0 method at creation; the engine's own setting is restored afterwards.
        crepe_mode = VocodeMode(config.extract_f0_mode) is VocodeMode.CREPE
        if crepe_mode:
            from . import crepe
            crepe.engine_with_model(self.engine)
            crepe.set_session_rate(fs, self.engine)
            prev_method = self.engine.f0_method
            self.engine.set_f0_method('crepe')
        if self._timing:
            prev = os.environ.get('RYK_STAGE_TIMES')
            os.environ['RYK_STAGE_TIMES'] = '1'
        try:
            self._sid = self.engine.session_create(cfg, voice=voice) if voice else self.engine.session_create(cfg)
        finally:
            if self._timing:
                if prev is None:
                    os.environ.pop('RYK_STAGE_TIMES', None)
                else:
                    os.environ['RYK_STAGE_TIMES'] = prev
            if crepe_mode:
                self.engine.set_f0_method(prev_method)
        if int(config.input_rate) != fs or int(config.output_rate) != fs:
            # the session resamples the sound card's chunks to fs and its output back to the card's rate on the device
            self.engine.session_set_input_rate(self._sid, int(config.input_rate))
            self.engine.session_set_output_rate(self._sid, int(config.output_rate))
            n_out_cap = self.engine.session_io_geometry(self._sid)['max_out']
        else:
            # capacity of one step's synthesizer output, as the session sizes it: (decode-window samples // block + 4) blocks
            rate = round(1000 / frame_period)
            hop = round(fs * frame_period / 1000)
            td = round(config.buffer_time * rate) + 2 * round(config.decode_extra_time * rate)
            n_out_cap = (td * hop // config.vocoder_buffer_size + 4) * config.vocoder_buffer_size
        if denoise is not None:
            self.engine.session_denoise(self._sid)
            self.engine.session_set_denoise(self._sid, float(denoise))
            if noise_profile is not None:
                self.engine.session_set_noise_profile(self._sid, noise_profile)
            if learn_noise is not None:
                self.engine.session_denoise_learn(self._sid, seconds=float(learn_noise))
        elif noise_profile is not None or learn_noise is not None:
            raise ValueError('noise_profile and learn_noise need denoise')
        self._echo = bool(echo_cancel)
        if self._echo:
            self.engine.session_echo_cancel(self._sid, taps=int(echo_taps), delay_ms=float(echo_delay_ms))
            self.engine.session_set_echo_suppression(self._sid, float(echo_suppression))
            self._played = numpy.zeros(config.in_audio_chunk, numpy.float32)   # the played stream not yet paired with an input chunk
        self._limiter = limiter is not None
        if self._limiter:             # the ceiling applies to the played level: the session's samples times output_scale
            self.engine.session_limiter(self._sid, lookahead_ms=float(limiter_lookahead_ms), hold_ms=float(limiter_hold_ms))
            self.engine.session_set_limiter(self._sid, float(limiter), gain=float(config.output_scale))
        if agc is not None:
            self.engine.session_agc(self._sid, float(agc), float(agc_max_gain_db), float(agc_gate_db))
        if pitch_correct is not None:
            self.engine.session_pitch_correct(self._sid)
            self.engine.session_set_pitch_correct(self._sid, **pitch_correct)
        if measure_f0 or follow_f0 is not None:
            self.engine.session_f0_measure(self._sid)
        if follow_f0 is not None:
            self.engine.session_f0_follow(self._sid, True, min_voiced_frames=int(follow_f0))
        if formant:
            self.engine.session_set_formant(self._sid, semitones=float(formant))
        self._scratch = numpy.empty(n_out_cap, dtype=numpy.float64)
        self._rid = self.engine.reblock_create(config.out_audio_chunk, n_out_cap, float(config.output_silent_threshold))
        self._drift, self._drift_ctl = None, None
        if drift is not None:           # the played stream's drift stage at the output rate: one out_audio_chunk per push
            self._drift = self.engine.drift_create(int(config.out_audio_chunk), float(drift_max_ppm))
            if drift == 'auto':
                self._drift_ctl = DriftController(int(config.output_rate), int(config.out_audio_chunk), max_ppm=float(drift_max_ppm))
            else:
                self.engine.drift_set(self._drift, float(drift))
        self._inflight: Deque[Tuple[Item, int, int, float]] = deque()      # (item, session ticket, re-blocker ticket, host time of put)
        self._done: Deque[Item] = deque()
        # audio-loop state (run.py:155-157)
        self._index_input = 0
        self._index_output = 0
        self._popped: List[Item] = []

    # ---- the session's f0 map -----------------------------------------------------------------------------------
    def set_f0_map(self, **kwargs) -> None:
        """Engine.session_set_f0_map for this stream (in_mean, in_std, target_mean, target_std, semitones): from the next chunk on."""
        self.engine.session_set_f0_map(self._sid, **kwargs)

    def set_formant(self, **kwargs) -> None:
        """Engine.session_set_formant for this stream (ratio or semitones): from the next chunk on."""
        self.engine.session_set_formant(self._sid, **kwargs)

    def set_voice(self, voice: int) -> None:
        """Convert into `voice` from the next chunk on, keeping the stream's state (no gap, no refill from silence).  The chunks in
        flight are finished first, in the new voice's place in the queue: their outputs stay queued for get / get_nowait in order.
        The f0 map becomes the new voice's, so a pitch offset set with set_f0_map must be set again afterwards; the formant ratio and
        the speaker statistics carry over."""
        while self._inflight:
            self._finish_one()
        self.engine.session_set_voice(self._sid, voice)

    def set_denoise(self, reduction_db: float) -> None:
        """Engine.session_set_denoise for this stream: the most the noise filter attenuates, from the next chunk on."""
        self.engine.session_set_denoise(self._sid, reduction_db)

    def noise_profile(self) -> Tuple[numpy.ndarray, int]:
        """(noise profile the next chunk uses, frames still to learn) of the stream's noise filter (needs denoise)."""
        return self.engine.session_noise_profile(self._sid)

    def set_echo_suppression(self, db: float) -> None:
        """Engine.session_set_echo_suppression for this stream: residual-echo suppression in dB, from the next chunk on."""
        self.engine.session_set_echo_suppression(self._sid, db)

    def echo_stats(self) -> Tuple[int, float]:
        """(frames, echo return loss enhancement in dB) of the last chunk put (needs echo_cancel)."""
        return self.engine.session_echo_stats(self._sid)

    def set_limiter(self, ceiling_db: float) -> None:
        """Engine.session_set_limiter for this stream: the ceiling of the played samples in dB of full scale, from the next chunk on
        (needs limiter)."""
        self.engine.session_set_limiter(self._sid, ceiling_db, gain=float(self.config.output_scale))

    def limiter_stats(self) -> Tuple[float, int]:
        """(largest gain reduction in dB, samples limited) of the last chunk put (needs limiter)."""
        return self.engine.session_limiter_stats(self._sid)

    def set_agc(self, target_db: Optional[float] = None, max_gain_db: Optional[float] = None, gate_db: Optional[float] = None) -> None:
        """Engine.session_set_agc for this stream: from the next chunk on; a None keeps that setting (needs agc)."""
        self.engine.session_set_agc(self._sid, target_db, max_gain_db, gate_db)

    def set_pitch_correct(self, **settings) -> None:
        """Engine.session_set_pitch_correct for this stream: key, scale, a4_hz, retune_ms and amount from the next chunk on; a missing
        one keeps its setting (needs pitch_correct)."""
        unknown = set(settings) - set(PITCH_CORRECT_KEYS)
        if unknown:
            raise ValueError(f'unknown pitch correction settings {sorted(unknown)}: use {", ".join(PITCH_CORRECT_KEYS)}')
        self.engine.session_set_pitch_correct(self._sid, **settings)

    def pitch_stats(self) -> Tuple[int, float, float]:
        """(voiced frames, mean and largest correction in cents) of the last chunk put (needs pitch_correct)."""
        return self.engine.session_pitch_stats(self._sid)

    def agc_stats(self) -> Tuple[float, float, int]:
        """(level in dB, -inf before any active block; gain in dB; active blocks of the last chunk) of the chunks put (needs agc)."""
        return self.engine.session_agc_stats(self._sid)

    def set_drift(self, ppm: float) -> None:
        """A fixed trim of the drift stage from the next chunk on (needs drift); in 'auto' mode it stops the controller."""
        self._need_drift()
        self.engine.drift_set(self._drift, float(ppm))
        self._drift_ctl = None

    def update_drift(self, backlog_samples: float) -> Optional[float]:
        """One reading of the output card's backlog in samples, taken after a chunk's write.  In 'auto' mode the controller turns it
        into the trim of the next chunk, which is returned; otherwise nothing changes and the trim in force (None without drift) is
        returned."""
        if self._drift is None:
            return None
        if self._drift_ctl is None:
            return self.engine.drift_get(self._drift)[0]
        ppm = self._drift_ctl.update(backlog_samples)
        self.engine.drift_set(self._drift, ppm)
        return ppm

    @property
    def drift_auto(self) -> bool:
        """whether a controller sets the drift stage's trim from the backlog readings update_drift gets"""
        return self._drift_ctl is not None

    def drift_stats(self) -> dict:
        """ppm and inc of the next chunk, the samples the stage consumed and produced, and whether the controller sets the trim."""
        self._need_drift()
        ppm, inc = self.engine.drift_get(self._drift)
        consumed, produced = self.engine.drift_stats(self._drift)
        return {'ppm': ppm, 'inc': inc, 'consumed': consumed, 'produced': produced, 'auto': self.drift_auto}

    def _need_drift(self) -> None:
        if self._drift is None:
            raise RuntimeError('the pipeline has no drift stage: create it with drift=PPM or drift=\'auto\'')

    def _drift_push(self, wave: numpy.ndarray) -> numpy.ndarray:
        return self.engine.drift_push(self._drift, wave).astype(numpy.float32)

    def measured_f0(self) -> Tuple[int, float, float]:
        """(voiced frames, mean, standard deviation) of the speaker's ln f0 over the chunks put so far (needs measure_f0)."""
        return self.engine.session_f0_measured(self._sid)

    # ---- queue_input_wave.put -------------------------------------------------------------------------------
    def put(self, item: Item) -> None:
        while len(self._inflight) >= self.depth:
            self._finish_one()
        ts = self.engine.session_submit(self._sid, numpy.asarray(item.item, dtype=numpy.float32))
        tr = self.engine.reblock_push_device(self._rid, self._sid)        # consumes the step's blocks in place, on its decode stream
        self._inflight.append((item, ts, tr, time.time()))

    def _finish_one(self) -> None:
        item, ts, tr, t_put = self._inflight.popleft()
        self.engine.session_collect(self._sid, ts, self._scratch)         # the raw blocks are not needed on the host
        _, chunk, _ = self.engine.reblock_collect(self._rid, tr)
        item.item = chunk                                                 # None: no chunk yet, or a silent one
        self._done.append(item)
        if self._timing:
            self._log_item(item.index, t_put)

    def _log_item(self, index: int, t_put: float) -> None:
        """DEBUG lines in the reference's format, one per stage logger: `<index>: <seconds>`; device time of the newest step's
        analysis (encode), gate + stage 1 + stage 2 (convert) and synthesis (decode), plus the host-side put -> collect latency."""
        try:
            st, en = self.engine.session_stage_times(self._sid)
            d = (en[-1] - st[-1]) * 1e-3
            enc, conv, dec = d[1], d[0] + d[2] + d[3], d[4]
        except Exception:                                                 # engines without stage timing (test doubles)
            enc = conv = dec = float('nan')
        self._loggers['encode'].debug(f'{index}: {enc}')
        self._loggers['convert'].debug(f'{index}: {conv}')
        self._loggers['decode'].debug(f'{index}: {dec} (put -> collect on the host: {time.time() - t_put})')

    # ---- queue_output_wave.get / get_nowait -----------------------------------------------------------------
    def get(self) -> Item:
        if not self._done:
            if not self._inflight:
                raise LookupError('nothing in flight')
            self._finish_one()
        return self._done.popleft()

    def _reap(self) -> None:
        """Move every in-flight item the device has already finished to `_done` without blocking (cudaEventQuery on the
        step's decode event and on the re-blocker event).  Chunks finish in submission order, so stop at the first busy one."""
        while self._inflight:
            _, ts, tr, _t = self._inflight[0]
            if not (self.engine.session_poll(self._sid, ts) and self.engine.reblock_poll(self._rid, tr)):
                break
            self._finish_one()

    def get_nowait(self) -> Optional[Item]:
        """An Item whose processing has finished, else None -- as soon as the device is done with it, like the reference's
        queue_output_wave.get_nowait() (run.py:176-182), not `depth` iterations later.  (The device finishes chunks in
        submission order; the reference's reorder buffer exists because its three processes finish out of order.)"""
        self._reap()
        return self._done.popleft() if self._done else None

    def flush(self) -> None:
        while self._inflight:
            self._finish_one()

    # ---- one iteration of the audio loop (run.py:160-199) -----------------------------------------------------
    def process(self, in_wave: numpy.ndarray, block: bool = False) -> numpy.ndarray:
        """in: in_audio_chunk float32 samples from the input device; out: out_audio_chunk float32 samples for the output
        device (zeros while nothing is ready, as the reference plays silence)."""
        c = self.config
        if self._echo:
            n = len(in_wave)
            far = self._played[:n]
            self._played = self._played[n:]
            self.engine.session_echo_reference(self._sid, numpy.concatenate([far, numpy.zeros(n - len(far), numpy.float32)]))
        self.put(Item(item=numpy.asarray(in_wave, dtype=numpy.float32) * c.input_scale, index=self._index_input))
        self._index_input += 1
        if block:
            self.flush()
        out_wave = self._next_output()
        if out_wave is None:
            out_wave = numpy.zeros(c.out_audio_chunk)
        out_wave = (out_wave * c.output_scale)[:c.out_audio_chunk].astype(numpy.float32)
        if self._echo:
            self._played = numpy.concatenate([self._played, out_wave])
        if self._drift is not None:
            out_wave = self._drift_push(out_wave)
        return out_wave

    def _next_output(self) -> Optional[numpy.ndarray]:
        """run.py:176-195: pop every finished item, take the ones whose index is next in order; silent items (None) are
        skipped; returns the first real chunk or None when nothing (more) is ready."""
        out_wave = None
        while True:
            while True:
                it = self.get_nowait()
                if it is None:
                    break
                self._popped.append(it)
            out_item = next((ii for ii in self._popped if ii.index == self._index_output), None)
            if out_item is None:
                break
            self._popped.remove(out_item)
            self._index_output += 1
            out_wave = out_item.item
            if out_wave is None:        # silence wave
                continue
            break
        return out_wave

    def drain(self) -> List[numpy.ndarray]:
        """End of a finite input (wav file): wait for everything in flight and return the output chunks not played yet, in
        order (the reference's loop never ends; a file-driven run must not lose the tail that is still in the pipeline).  With drift the
        chunks go through the drift stage and a last item flushes the 16 samples it holds: the played stream ends here."""
        c = self.config
        self.flush()
        outs: List[numpy.ndarray] = []
        while self._done or self._popped:
            w = self._next_output()
            if w is None:
                break
            outs.append((w * c.output_scale)[:c.out_audio_chunk].astype(numpy.float32))
        if self._drift is not None:
            outs = [self._drift_push(w) for w in outs] + [self._drift_push(numpy.zeros(DRIFT_HALF_WIDTH, numpy.float32))]
        return outs

    # ---- moving the stream (DESIGN.md §4k) ----------------------------------------------------------------------
    def snapshot(self) -> bytes:
        """The whole stream state as one blob: the session's, the re-blocker's and the pipeline's host state (the next item index,
        the echo far-end queue, input_scale and output_scale; with drift the drift stage's blob and the controller's state).  Only a
        drained pipeline can be snapshotted: nothing in flight and every finished item taken (`drain`)."""
        if self._inflight or self._done or self._popped or self._index_output != self._index_input:
            raise RuntimeError('the pipeline has chunks in flight or outputs not taken: drain() it before a snapshot')
        host = {'index': self._index_input, 'input_scale': float(self.config.input_scale),
                'output_scale': float(self.config.output_scale), 'echo': self._echo, 'limiter': self._limiter}
        if self._drift is not None:
            host['drift'] = {'controller': None if self._drift_ctl is None else self._drift_ctl.state()}
        return pack_pipeline(self.engine.session_snapshot(self._sid), self.engine.reblock_snapshot(self._rid), host,
                             self._played if self._echo else None,
                             None if self._drift is None else self.engine.drift_snapshot(self._drift))

    @classmethod
    def restore(cls, blob: bytes, config: Config, engine: Optional[Engine] = None, voice: int = 0, depth: int = 3,
                acoustic_param=None) -> 'RealtimePipeline':
        """The pipeline a snapshot was taken of, continued on `engine` (another engine or GPU too) and converting into `voice`: the same
        items give the same outputs bit for bit.  The models of `voice` must be loaded into `engine`.  Refused (ValueError) when the
        blob's recorded configuration does not match `config` and the frame period of `acoustic_param`, as the constructor takes them."""
        parts = unpack_pipeline(blob)
        check_pipeline_config(parts, config, acoustic_param)
        self = cls.__new__(cls)
        self.config = config
        self.engine = engine or default_engine()
        if parts['session_config']['f0_method'] == 2:
            # CREPE: the same model and resampler taps a pipeline created in CREPE mode loads (RYK_CREPE_MODEL when none is loaded)
            from . import crepe
            crepe.engine_with_model(self.engine)
            crepe.set_session_rate(int(parts['session_config']['cfg']['fs']), self.engine)
        self.depth = max(1, min(int(depth), 5))
        self._loggers = {k: logging.getLogger(k) for k in ('encode', 'convert', 'decode')}
        self._timing = False
        self._sid = self.engine.session_restore(parts['session'], voice=voice)
        try:
            self._rid = self.engine.reblock_restore(parts['reblock'])
        except Exception:
            self.engine.session_destroy(self._sid)
            raise
        host = parts['host']
        self._drift, self._drift_ctl = None, None
        if parts['drift'] is not None:
            try:
                self._drift = self.engine.drift_restore(parts['drift'])
            except Exception:
                self.engine.reblock_destroy(self._rid)
                self.engine.session_destroy(self._sid)
                raise
            ctl = host['drift']['controller']
            self._drift_ctl = None if ctl is None else DriftController.from_state(ctl)
        self._echo, self._limiter = bool(host['echo']), bool(host['limiter'])
        if self._echo:
            self._played = parts['played']
        self._scratch = numpy.empty(self.engine.session_io_geometry(self._sid)['max_out'], dtype=numpy.float64)
        self._inflight = deque()
        self._done = deque()
        self._index_input = self._index_output = int(host['index'])
        self._popped = []
        return self

    def close(self) -> None:
        if self._sid is not None:
            self.flush()
            self.engine.reblock_destroy(self._rid)
            if self._drift is not None:
                self.engine.drift_destroy(self._drift)
                self._drift = None
            self.engine.session_destroy(self._sid)
            self._sid = None


# ---- the pipeline blob: the snapshot container (snapshot.py) of kind 'pipeline' ------------------------------------------------------
# SESS: the session's blob, RBLK: the re-blocker's blob, PIPE: the pipeline's host state as JSON, FARQ: the echo far-end queue (float32),
# DRFT: the drift stage's blob.
def pack_pipeline(session: bytes, reblock: bytes, host: dict, played: Optional[numpy.ndarray], drift: Optional[bytes] = None) -> bytes:
    from .snapshot import pack
    sections = [('SESS', session), ('RBLK', reblock), ('PIPE', json.dumps(host, sort_keys=True).encode('utf-8'))]
    if played is not None:
        sections.append(('FARQ', numpy.ascontiguousarray(played, dtype=numpy.float32).tobytes()))
    if drift is not None:
        sections.append(('DRFT', drift))
    return pack('pipeline', sections)


def unpack_pipeline(blob: bytes) -> dict:
    """{'session', 'reblock': blobs, 'host': dict, 'played': float32 array or None, 'drift': blob or None, 'session_config',
    'reblock_config': the configurations the two blobs record}; raises ValueError for a blob that is not a pipeline snapshot."""
    from .engine import RykError, describe_snapshot
    from .snapshot import unpack
    try:
        kind, sec = unpack(blob)
        if kind != 'pipeline' or not {'SESS', 'RBLK', 'PIPE'} <= set(sec):
            raise ValueError('not a pipeline snapshot')
        host = json.loads(sec['PIPE'].decode('utf-8'))
        ds, dr = describe_snapshot(sec['SESS']), describe_snapshot(sec['RBLK'])
        dd = describe_snapshot(sec['DRFT']) if 'DRFT' in sec else None
    except RykError as exc:
        raise ValueError(f'not a usable pipeline snapshot: {exc}') from exc
    if ds['kind'] != 'session' or dr['kind'] != 'reblock' or (dd is not None and dd['kind'] != 'drift'):
        raise ValueError('not a pipeline snapshot')
    played = numpy.frombuffer(sec['FARQ'], dtype=numpy.float32).copy() if 'FARQ' in sec else None
    if bool(host.get('echo')) != (played is not None):
        raise ValueError('malformed pipeline snapshot: the echo far-end queue')
    if ('drift' in host) != (dd is not None):
        raise ValueError('malformed pipeline snapshot: the drift stage')
    return {'session': sec['SESS'], 'reblock': sec['RBLK'], 'host': host, 'played': played, 'drift': sec.get('DRFT'),
            'session_config': ds['config'], 'reblock_config': dr['config']}


def check_pipeline_config(parts: dict, config: Config, acoustic_param=None) -> None:
    """Refuse (ValueError, listing every difference) a pipeline snapshot whose recorded configuration is not what `config` and the
    model's `acoustic_param` make."""
    sc, rc, host = parts['session_config'], parts['reblock_config'], parts['host']
    cfg = sc['cfg']
    fs = int(cfg['fs'])
    crepe = VocodeMode(config.extract_f0_mode) is VocodeMode.CREPE
    want = [
        ('model frame_period', cfg['frame_period_ms'], model_frame_period(acoustic_param)),
        ('buffer_time', cfg['buffer_time'], float(config.buffer_time)),
        ('encode_extra_time', cfg['encode_extra_time'], float(config.encode_extra_time)),
        ('convert_extra_time', cfg['convert_extra_time'], float(config.convert_extra_time)),
        ('decode_extra_time', cfg['decode_extra_time'], float(config.decode_extra_time)),
        ('input_silent_threshold', cfg['threshold_db'], float(config.input_silent_threshold)),
        ('vocoder_buffer_size', cfg['vocoder_buffer_size'], int(config.vocoder_buffer_size)),
        ('input_rate', sc['in_rate'] or fs, int(config.input_rate)),
        ('output_rate', sc['out_rate'] or fs, int(config.output_rate)),
        ('extract_f0_mode crepe', sc['f0_method'] == 2, crepe),
        ('out_audio_chunk', rc['out_audio_chunk'], int(config.out_audio_chunk)),
        ('output_silent_threshold', rc['threshold_db'], float(config.output_silent_threshold)),
        ('input_scale', host.get('input_scale'), float(config.input_scale)),
        ('output_scale', host.get('output_scale'), float(config.output_scale)),
    ]
    bad = [f'{name}: recorded {got}, config {exp}' for name, got, exp in want if got != exp]
    if bad:
        raise ValueError('the snapshot was taken with another configuration: ' + '; '.join(bad))
