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
import logging
import os
import time
from collections import deque
from typing import Any, Deque, List, Optional, Tuple

import numpy

from .config import Config, VocodeMode
from .engine import Engine, SessionConfig, default_engine


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


class RealtimePipeline(object):
    """encode_worker | convert_worker | decode_worker of one audio stream as one device-resident session.

    The models must already be loaded into `engine` (YukarinConverter.make_yukarin_converter does that for voice 0,
    models.load_voice for any voice); the session converts into `voice`.  `depth` chunks may be in flight (the reference's queues
    are unbounded; the session keeps up to 5 steps in flight).

    `measure_f0=True` keeps running statistics of the speaker's log-f0 on the device (`measured_f0`); `follow_f0=N` (implies
    measuring) also makes them the input side of the session's f0 map once N voiced frames are counted.  `set_f0_map` changes the
    map between chunks."""

    def __init__(self, config: Config, acoustic_param=None, engine: Optional[Engine] = None, depth: int = 3, voice: int = 0,
                 measure_f0: bool = False, follow_f0: Optional[int] = None):
        self.config = config
        self.engine = engine or default_engine()
        p = acoustic_param
        # analysis, the U-Nets and synthesis run at the models' rate; the sound card's rates are the session's device rates
        fs = int(getattr(p, 'sampling_rate', 24000))
        cfg = SessionConfig(
            fs=fs, frame_period_ms=float(config.frame_period),
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
            rate = round(1000 / float(config.frame_period))
            hop = round(fs * float(config.frame_period) / 1000)
            td = round(config.buffer_time * rate) + 2 * round(config.decode_extra_time * rate)
            n_out_cap = (td * hop // config.vocoder_buffer_size + 4) * config.vocoder_buffer_size
        if measure_f0 or follow_f0 is not None:
            self.engine.session_f0_measure(self._sid)
        if follow_f0 is not None:
            self.engine.session_f0_follow(self._sid, True, min_voiced_frames=int(follow_f0))
        self._scratch = numpy.empty(n_out_cap, dtype=numpy.float64)
        self._rid = self.engine.reblock_create(config.out_audio_chunk, n_out_cap, float(config.output_silent_threshold))
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
        self.put(Item(item=numpy.asarray(in_wave, dtype=numpy.float32) * c.input_scale, index=self._index_input))
        self._index_input += 1
        if block:
            self.flush()
        out_wave = self._next_output()
        if out_wave is None:
            out_wave = numpy.zeros(c.out_audio_chunk)
        out_wave = out_wave * c.output_scale
        return out_wave[:c.out_audio_chunk].astype(numpy.float32)

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
        order (the reference's loop never ends; a file-driven run must not lose the tail that is still in the pipeline)."""
        c = self.config
        self.flush()
        outs: List[numpy.ndarray] = []
        while self._done or self._popped:
            w = self._next_output()
            if w is None:
                break
            outs.append((w * c.output_scale)[:c.out_audio_chunk].astype(numpy.float32))
        return outs

    def close(self) -> None:
        if self._sid is not None:
            self.flush()
            self.engine.reblock_destroy(self._rid)
            self.engine.session_destroy(self._sid)
            self._sid = None
