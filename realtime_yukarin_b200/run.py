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
from .models import write_f0_statistics
from .worker import RealtimePipeline


def audio_loop(pipeline: RealtimePipeline, read_chunk: Callable[[], Optional[numpy.ndarray]],
               write_chunk: Callable[[numpy.ndarray], None], max_chunks: Optional[int] = None) -> int:
    """run.py:152-199: read one input chunk, queue it, play whatever output is ready (zeros otherwise).  Returns the number of
    chunks processed; stops when `read_chunk` returns None (end of a wav file) or after `max_chunks`."""
    n = 0
    while max_chunks is None or n < max_chunks:
        in_wave = read_chunk()
        if in_wave is None:
            break
        write_chunk(pipeline.process(in_wave))
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


def run(config_path: Path, wav_in: Optional[Path] = None, wav_out: Optional[Path] = None, max_chunks: Optional[int] = None,
        engine=None, depth: int = 3, measure_input_statistics: Optional[Path] = None, follow_input_f0: Optional[int] = None,
        pitch: float = 0.0) -> int:
    """`measure_input_statistics`: measure the speaker's log-f0 statistics during the run and write them to this file at the end;
    `follow_input_f0`: convert with the measured statistics once this many voiced frames are counted; `pitch`: semitones added to
    the target voice's mean f0."""
    logger = logging.getLogger('root')
    logger.info('model loading...')
    config = Config.from_yaml(config_path)
    converter = YukarinConverter.make_yukarin_converter(
        input_statistics_path=config.input_statistics_path, target_statistics_path=config.target_statistics_path,
        stage1_model_path=config.stage1_model_path, stage1_config_path=config.stage1_config_path,
        stage2_model_path=config.stage2_model_path, stage2_config_path=config.stage2_config_path)
    pipeline = RealtimePipeline(config, acoustic_param=converter.acoustic_converter.config.dataset.acoustic_param, engine=engine, depth=depth,
                                measure_f0=measure_input_statistics is not None, follow_f0=follow_input_f0)
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
        return audio_loop(pipeline, lambda: numpy.frombuffer(stream_in.read(config.in_audio_chunk), dtype=numpy.float32),
                          lambda w: stream_out.write(w.astype(numpy.float32).tobytes()), max_chunks)
    finally:
        try:
            if measure_input_statistics is not None:
                pipeline.flush()
                save_measured_statistics(pipeline, measure_input_statistics)
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
                        help='shift the converted f0 by this many semitones (the spectral envelope is not moved)')
    return parser


def main(argv: Optional[Iterable[str]] = None) -> None:
    args = make_parser().parse_args(argv)
    run(config_path=args.config_path, wav_in=args.wav_in, wav_out=args.wav_out, max_chunks=args.max_chunks,
        measure_input_statistics=args.measure_input_statistics, follow_input_f0=args.follow_input_f0, pitch=args.pitch)


if __name__ == '__main__':
    main()
