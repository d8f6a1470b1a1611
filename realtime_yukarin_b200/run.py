"""`python -m realtime_yukarin_b200.run --config_path config.yaml` -- the reference's run.py (run.py:22-199) on one H100.

Same config file (config.yaml), same model loading (YukarinConverter.make_yukarin_converter) and the same audio loop; the
three worker processes and their queues (run.py:58-93) are one device-resident session (worker.RealtimePipeline).

Audio I/O: PyAudio when it is installed (as in the reference: float32 mono, frames_per_buffer = in / out_audio_chunk, devices
picked by name, run.py:98-139).  `--wav_in / --wav_out` replace the microphone / speaker by wav files -- the loop body is
identical -- which is also how the loop is exercised in tests (no audio hardware on a GPU box).
"""
import argparse
import logging
import signal
import sys
from pathlib import Path
from typing import Callable, Iterable, Optional

import numpy

from . import wave_io
from .config import Config
from .converter import YukarinConverter
from .engine import pitch_key, pitch_scale
from .models import write_f0_statistics
from .worker import RealtimePipeline, pitch_settings, unpack_pipeline


def audio_loop(pipeline: RealtimePipeline, read_chunk: Callable[[], Optional[numpy.ndarray]],
               write_chunk: Callable[[numpy.ndarray], None], max_chunks: Optional[int] = None,
               backlog: Optional[Callable[[], float]] = None) -> int:
    """run.py:152-199: read one input chunk, queue it, play whatever output is ready (zeros otherwise).  Returns the number of
    chunks processed; stops when `read_chunk` returns None (end of a wav file) or after `max_chunks`.  `backlog`: read the output
    card's queue after each write and hand it to the pipeline's drift controller (RealtimePipeline.update_drift)."""
    n = 0
    while max_chunks is None or n < max_chunks:
        in_wave = read_chunk()
        if in_wave is None:
            break
        write_chunk(pipeline.process(in_wave))
        if backlog is not None:
            pipeline.update_drift(backlog())
        n += 1
    return n


def _find_device(audio, name: Optional[str], kind: str) -> int:
    if name is None:
        info = audio.get_default_input_device_info() if kind == 'input' else audio.get_default_output_device_info()
        return info['index']
    for i in range(audio.get_device_count()):
        if name in str(audio.get_device_info_by_index(i)['name']):
            return i
    raise ValueError(f'{kind} device not found')


def save_measured_statistics(pipeline: RealtimePipeline, path: Path) -> bool:
    """Write the speaker's log-f0 statistics the session measured to `path` (an input_statistics file) and print them; nothing is
    written when the input held fewer than two voiced frames or a single pitch."""
    n, mean, std = pipeline.measured_f0()
    print(f'measured log-f0 over {n} voiced frames: mean {mean:.6f} ({numpy.exp(mean):.1f} Hz), std {std:.6f}')
    if n < 2 or not std > 0:
        print(f'not enough voiced input for statistics: {path} was not written')
        return False
    write_f0_statistics(path, mean, std * std)
    print(f'wrote {path}')
    return True


def save_noise_profile_file(pipeline: RealtimePipeline, path: Path) -> None:
    """Write the noise profile the stream's filter uses now to `path` (.npy, 257 float64 powers) for a later --noise_profile."""
    phi, left = pipeline.noise_profile()
    if left:
        print(f'the noise profile was still being learned ({left} frames to go): {path} holds the profile in use before it')
    numpy.save(path, phi)
    print(f'wrote {path}')


def save_state_file(pipeline: RealtimePipeline, path: Path) -> None:
    """Write the stream state of `pipeline` to `path` for a later --load_state (after taking the outputs still in flight)."""
    pipeline.drain()
    Path(path).write_bytes(pipeline.snapshot())
    print(f'wrote {path}')


# options that set up the stream's stages, with the values that leave them off: a state file brings its own stages
_STAGE_OPTIONS = {'follow_input_f0': None, 'pitch': 0.0, 'formant': 0.0, 'denoise': None, 'noise_profile': None, 'learn_noise': None,
                  'echo_cancel': None, 'echo_delay': 0.0, 'echo_suppression': 0.0, 'limit': None, 'limit_lookahead': None,
                  'limit_hold': None, 'agc': None, 'agc_max_gain': None, 'agc_gate': None, 'drift_ppm': None, 'drift': None,
                  'autotune': None, 'retune_ms': None, 'autotune_amount': None}


def autotune_settings(autotune: str, retune_ms: Optional[float] = None, amount: Optional[float] = None) -> dict:
    """--autotune KEY[:SCALE] (SCALE: major when missing, minor, chromatic or a 12-bit mask such as 0xab5) with --retune_ms (50 when
    None) and --autotune_amount (1 when None), as RealtimePipeline(pitch_correct=...) takes them."""
    key, _, scale = str(autotune).partition(':')
    scale = scale.strip() or 'major'
    try:
        scale = int(scale, 0)
    except ValueError:
        pass
    return dict(key=pitch_key(key), scale=pitch_scale(scale), retune_ms=50.0 if retune_ms is None else float(retune_ms),
                amount=1.0 if amount is None else float(amount))


def run(config_path: Path, wav_in: Optional[Path] = None, wav_out: Optional[Path] = None, max_chunks: Optional[int] = None,
        engine=None, depth: int = 3, measure_input_statistics: Optional[Path] = None, follow_input_f0: Optional[int] = None,
        pitch: float = 0.0, formant: float = 0.0, denoise: Optional[float] = None, noise_profile: Optional[Path] = None,
        learn_noise: Optional[float] = None, save_noise_profile: Optional[Path] = None, echo_cancel: Optional[int] = None,
        echo_delay: float = 0.0, echo_suppression: float = 0.0, limit: Optional[float] = None,
        limit_lookahead: Optional[float] = None, limit_hold: Optional[float] = None, agc: Optional[float] = None,
        agc_max_gain: Optional[float] = None, agc_gate: Optional[float] = None, save_state: Optional[Path] = None,
        load_state: Optional[Path] = None, drift_ppm: Optional[float] = None, drift: Optional[float] = None,
        autotune: Optional[str] = None, retune_ms: Optional[float] = None, autotune_amount: Optional[float] = None) -> int:
    """`measure_input_statistics`: measure the speaker's log-f0 statistics during the run and write them to this file at the end;
    `follow_input_f0`: convert with the measured statistics once this many voiced frames are counted; `pitch`: semitones added to
    the target voice's mean f0; `formant`: semitones by which the converted spectral envelope moves; `denoise`: filter the input's
    noise ahead of the analysis with at most this many dB of attenuation, with the profile in `noise_profile` (.npy) or one learned from
    the first `learn_noise` seconds of input, and write the profile in use to `save_noise_profile` at the end; `echo_cancel`: cancel the
    echo of the played output in the input with a filter of this many 128-sample frames after a bulk delay of `echo_delay` ms, followed
    by `echo_suppression` dB of residual-echo suppression; `limit`: keep the played output under this ceiling (dB of full scale) with a
    look-ahead peak limiter of `limit_lookahead` ms (the output delay grows by as much; 5 when None) holding each reduction for
    `limit_hold` ms (50 when None); `agc`: bring the speaker's level to this target (dB of full scale) ahead of the analysis with at most
    `agc_max_gain` dB of gain (20 when None), counting only input louder than `agc_gate` dB (-50 when None); `save_state`: write the
    stream state (worker.RealtimePipeline.snapshot) to this file when the audio loop ends; `load_state`: continue the stream such a file
    holds (learned noise profile, echo path, AGC level, f0 statistics and every setting), refused when it was written with another
    configuration and with the options that set up stages, which the file brings; --save_noise_profile and --measure_input_statistics
    then need the stage in the file; `drift_ppm`: play the output (1 + drift_ppm 1e-6) times as long through the drift stage, a fixed trim
    for an output sound card whose clock runs that much fast; `drift`: let a controller find the trim, up to +-drift ppm, from the output
    card's backlog (live audio only: with wav files there is no second clock); `autotune`: 'KEY[:SCALE]', pull each converted note
    toward the nearest note of that scale (major when no SCALE is given) with a retune time of `retune_ms` (50 when None; 0 snaps) and
    `autotune_amount` of the correction (1 when None)."""
    state = None
    if load_state is not None:
        values = locals()
        given = [name for name, off in _STAGE_OPTIONS.items() if values[name] != off]
        if given:
            raise ValueError('--load_state brings the stages of the saved stream: drop ' + ', '.join('--' + n for n in given))
        state = Path(load_state).read_bytes()
        recorded = unpack_pipeline(state)['session_config']
        if save_noise_profile is not None and not recorded['denoise']:
            raise ValueError('--save_noise_profile needs noise suppression, which the stream in --load_state does not run')
        if measure_input_statistics is not None and not recorded['f0_measure']:
            raise ValueError('--measure_input_statistics needs f0 measuring, which the stream in --load_state does not run')
    if drift is not None and drift_ppm is not None:
        raise ValueError('--drift and --drift_ppm exclude each other: the controller sets the trim, or --drift_ppm fixes it')
    if drift is not None and wav_in is not None:
        raise ValueError('--drift needs live audio: with --wav_in there is no second clock to follow (--drift_ppm sets a fixed trim)')
    if autotune is None and (retune_ms is not None or autotune_amount is not None):
        raise ValueError('--retune_ms and --autotune_amount need --autotune')
    pitch_correct = None if autotune is None else pitch_settings(autotune_settings(autotune, retune_ms, autotune_amount))
    if agc is None and (agc_max_gain is not None or agc_gate is not None):
        raise ValueError('--agc_max_gain and --agc_gate need --agc')
    if limit is None and (limit_lookahead is not None or limit_hold is not None):
        raise ValueError('--limit_lookahead and --limit_hold need --limit')
    if echo_cancel is None and (echo_delay or echo_suppression):
        raise ValueError('--echo_delay and --echo_suppression need --echo_cancel')
    if denoise is None and (noise_profile is not None or learn_noise is not None or (save_noise_profile is not None and state is None)):
        raise ValueError('--noise_profile, --learn_noise and --save_noise_profile need --denoise')
    logger = logging.getLogger('root')
    logger.info('model loading...')
    config = Config.from_yaml(config_path)
    converter = YukarinConverter.make_yukarin_converter(
        input_statistics_path=config.input_statistics_path, target_statistics_path=config.target_statistics_path,
        stage1_model_path=config.stage1_model_path, stage1_config_path=config.stage1_config_path,
        stage2_model_path=config.stage2_model_path, stage2_config_path=config.stage2_config_path)
    if load_state is not None:
        pipeline = RealtimePipeline.restore(state, config, engine=engine, depth=depth,
                                            acoustic_param=converter.acoustic_converter.config.dataset.acoustic_param)
    else:
        pipeline = RealtimePipeline(config, acoustic_param=converter.acoustic_converter.config.dataset.acoustic_param, engine=engine, depth=depth,
                                measure_f0=measure_input_statistics is not None, follow_f0=follow_input_f0, formant=formant,
                                denoise=denoise, noise_profile=None if noise_profile is None else numpy.load(noise_profile),
                                learn_noise=learn_noise, echo_cancel=echo_cancel is not None,
                                echo_taps=32 if echo_cancel is None else echo_cancel, echo_delay_ms=echo_delay,
                                echo_suppression=echo_suppression, limiter=limit,
                                limiter_lookahead_ms=5.0 if limit_lookahead is None else limit_lookahead,
                                limiter_hold_ms=50.0 if limit_hold is None else limit_hold, agc=agc,
                                agc_max_gain_db=20.0 if agc_max_gain is None else agc_max_gain,
                                agc_gate_db=-50.0 if agc_gate is None else agc_gate,
                                drift='auto' if drift is not None else drift_ppm,
                                drift_max_ppm=drift if drift is not None else max(500.0, abs(drift_ppm or 0.0)),
                                pitch_correct=pitch_correct)
    try:
        if pitch:
            pipeline.set_f0_map(semitones=pitch)
        if wav_in is not None:
            wave = wave_io.load_wave(wav_in, config.input_rate, engine=engine).wave
            pos = [0]
            out_chunks = []

            def read_chunk():
                a = pos[0]
                if a + config.in_audio_chunk > len(wave):
                    return None
                pos[0] = a + config.in_audio_chunk
                return wave[a:a + config.in_audio_chunk]

            n = audio_loop(pipeline, read_chunk, out_chunks.append, max_chunks)
            out_chunks.extend(pipeline.drain())      # chunks still in flight when the file ended
            if wav_out is not None:
                wave_io.write_wav(wav_out, numpy.concatenate(out_chunks) if out_chunks else numpy.zeros(0, numpy.float32), config.output_rate)
            return n
        try:
            import pyaudio
        except ImportError as exc:
            raise RuntimeError('PyAudio is not installed: use --wav_in / --wav_out, or install it for live audio') from exc
        audio = pyaudio.PyAudio()
        stream_in = audio.open(format=pyaudio.paFloat32, channels=1, rate=config.input_rate, frames_per_buffer=config.in_audio_chunk,
                               input=True, input_device_index=_find_device(audio, config.input_device_name, 'input'))
        stream_out = audio.open(format=pyaudio.paFloat32, channels=1, rate=config.output_rate, frames_per_buffer=config.out_audio_chunk,
                                output=True, output_device_index=_find_device(audio, config.output_device_name, 'output'))
        signal.signal(signal.SIGINT, lambda s, f: sys.exit(0))
        logger.debug('audio loop')
        # the controller regulates the backlog to a set-point it learns, so the free space of the output buffer, negated, serves as its fill
        backlog = (lambda: -float(stream_out.get_write_available())) if pipeline.drift_auto else None
        return audio_loop(pipeline, lambda: numpy.frombuffer(stream_in.read(config.in_audio_chunk), dtype=numpy.float32),
                          lambda w: stream_out.write(w.astype(numpy.float32).tobytes()), max_chunks, backlog=backlog)
    finally:
        try:
            if measure_input_statistics is not None:
                pipeline.flush()
                save_measured_statistics(pipeline, measure_input_statistics)
            if save_noise_profile is not None:
                pipeline.flush()
                save_noise_profile_file(pipeline, save_noise_profile)
            if save_state is not None:                # here too when Ctrl-C ends a live loop (SystemExit)
                save_state_file(pipeline, save_state)
        finally:
            pipeline.close()


def make_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser()
    parser.add_argument('--config_path', type=Path, default=Path('./config.yaml'))
    parser.add_argument('--wav_in', type=Path, default=None, help='feed this wav file instead of the input device')
    parser.add_argument('--wav_out', type=Path, default=None, help='with --wav_in: write the played chunks to this wav file')
    parser.add_argument('--max_chunks', type=int, default=None)
    parser.add_argument('--measure_input_statistics', type=Path, default=None, metavar='OUT.npy',
                        help="measure the log-f0 statistics of the speaker on the input during the run and write them to this file "
                             "when it ends: the file config.yaml's input_statistics_path expects")
    parser.add_argument('--follow_input_f0', type=int, nargs='?', const=200, default=None, metavar='MIN_FRAMES',
                        help='convert f0 with the statistics measured on the input so far instead of input_statistics_path, once '
                             'MIN_FRAMES voiced 5 ms frames are counted (default 200)')
    parser.add_argument('--pitch', type=float, default=0.0, metavar='SEMITONES',
                        help='shift the converted f0 by this many semitones (the spectral envelope is not moved: see --formant)')
    parser.add_argument('--formant', type=float, default=0.0, metavar='SEMITONES',
                        help='move the converted spectral envelope (the formants) by this many semitones, -12 to 12; with --pitch '
                             'by the same amount the voice sounds like a different speaker rather than the same one at another pitch')
    parser.add_argument('--denoise', type=float, default=None, metavar='DB',
                        help='suppress the noise of the input ahead of the analysis, attenuating by at most DB (0-40; 20 is a good '
                             'start); the noise profile comes from --noise_profile or --learn_noise (without one the input passes unchanged)')
    parser.add_argument('--noise_profile', type=Path, default=None, metavar='IN.npy', help='with --denoise: the noise profile to use')
    parser.add_argument('--learn_noise', type=float, default=None, metavar='SECONDS',
                        help='with --denoise: learn the noise profile from the first SECONDS of input (stay quiet meanwhile; 1 s is enough)')
    parser.add_argument('--save_noise_profile', type=Path, default=None, metavar='OUT.npy',
                        help='with --denoise: write the noise profile in use to this file when the run ends, for --noise_profile')
    parser.add_argument('--echo_cancel', type=int, nargs='?', const=32, default=None, metavar='TAPS',
                        help='cancel the echo of the played output that the microphone picks up (speakers instead of headphones), with '
                             'a filter of TAPS frames of 128 samples at the model rate (1-64, default 32: 170 ms at 24 kHz)')
    parser.add_argument('--echo_delay', type=float, default=0.0, metavar='MS',
                        help='with --echo_cancel: the bulk delay of the echo path ahead of the filter, in ms (up to 256 frames)')
    parser.add_argument('--echo_suppression', type=float, default=0.0, metavar='DB',
                        help='with --echo_cancel: suppress the residual echo by at most DB (0-40; 0 keeps the linear canceller)')
    parser.add_argument('--limit', type=float, nargs='?', const=-1.0, default=None, metavar='CEILING_DB',
                        help='keep the played output (after output_scale) under CEILING_DB of full scale with a look-ahead peak '
                             'limiter on the GPU (-24 to 0, default -1), so that loud syllables do not clip at the sound card')
    parser.add_argument('--limit_lookahead', type=float, default=None, metavar='MS',
                        help='with --limit: look-ahead of the limiter in ms (0.5-10, default 5); the output delay grows by as much')
    parser.add_argument('--limit_hold', type=float, default=None, metavar='MS',
                        help='with --limit: how long a gain reduction is held before it ramps back, in ms (0-500, default 50)')
    parser.add_argument('--agc', type=float, nargs='?', const=-26.0, default=None, metavar='TARGET_DB',
                        help='bring the speaker to TARGET_DB (mean square, dB of full scale; -40 to -6, default -26) ahead of the '
                             'analysis with an automatic gain control on the GPU, after input_scale, echo cancellation and noise suppression')
    parser.add_argument('--agc_max_gain', type=float, default=None, metavar='DB',
                        help='with --agc: the most the gain control amplifies or attenuates, in dB (0-30, default 20)')
    parser.add_argument('--agc_gate', type=float, default=None, metavar='DB',
                        help='with --agc: blocks of input at or under this level (dB of full scale, -80 to -20, default -50) leave '
                             'the level and the gain as they are')
    parser.add_argument('--drift_ppm', type=float, default=None, metavar='PPM',
                        help='play the output (1 + PPM 1e-6) times as long (a fixed trim, -2000 to 2000), for an output sound card whose '
                             'clock runs PPM ppm fast against the input card\'s; works with --wav_in too')
    parser.add_argument('--drift', type=float, nargs='?', const=500.0, default=None, metavar='MAX_PPM',
                        help='follow the clock difference of the input and output sound cards: a controller trims the played stream '
                             'by up to MAX_PPM (default 500, at most 2000) from the output card\'s backlog, so a long session neither '
                             'underruns nor falls behind (live audio only)')
    parser.add_argument('--autotune', type=str, default=None, metavar='KEY[:SCALE]',
                        help='pull each converted note toward the nearest note of a scale on the GPU: KEY is a note name (C, F#, Bb) '
                             'or 0-11, SCALE major (default), minor, chromatic or a 12-bit mask of pitch classes above the key')
    parser.add_argument('--retune_ms', type=float, default=None, metavar='MS',
                        help='with --autotune: how fast a note is pulled to the scale, in ms (0-1000, default 50; 0 snaps at once)')
    parser.add_argument('--autotune_amount', type=float, default=None, metavar='A',
                        help='with --autotune: the share of the correction applied (0-1, default 1)')
    parser.add_argument('--save_state', type=Path, default=None, metavar='OUT.state',
                        help='when the audio loop ends, write the stream state (learned noise profile, echo path, AGC level, f0 '
                             'statistics, settings) to this file for --load_state')
    parser.add_argument('--load_state', type=Path, default=None, metavar='IN.state',
                        help='continue the stream a --save_state file holds; the file must come from the same configuration and '
                             'brings its own stages, so the stage options are refused with it')
    return parser


def main(argv: Optional[Iterable[str]] = None) -> None:
    args = make_parser().parse_args(argv)
    run(config_path=args.config_path, wav_in=args.wav_in, wav_out=args.wav_out, max_chunks=args.max_chunks,
        measure_input_statistics=args.measure_input_statistics, follow_input_f0=args.follow_input_f0, pitch=args.pitch,
        formant=args.formant, denoise=args.denoise, noise_profile=args.noise_profile, learn_noise=args.learn_noise,
        save_noise_profile=args.save_noise_profile, echo_cancel=args.echo_cancel, echo_delay=args.echo_delay,
        echo_suppression=args.echo_suppression, limit=args.limit, limit_lookahead=args.limit_lookahead, limit_hold=args.limit_hold,
        agc=args.agc, agc_max_gain=args.agc_max_gain, agc_gate=args.agc_gate, save_state=args.save_state, load_state=args.load_state,
        drift_ppm=args.drift_ppm, drift=args.drift, autotune=args.autotune, retune_ms=args.retune_ms,
        autotune_amount=args.autotune_amount)


if __name__ == '__main__':
    main()
