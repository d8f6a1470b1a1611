"""wav I/O and sample-rate conversion next to the hot path (SURVEY 8(f) rank 3; check.py:78-81 `librosa.load(path, sr=input_rate)`,
check.py:110-112 `librosa.output.write_wav(path, wave.astype(float32), output_rate)`).

librosa / resampy are not available here (SURVEY 8c), so the resampler is the polyphase FIR method of
scipy.signal.resample_poly (Kaiser beta = 5 windowed sinc, half length 10 * max(up, down), zero-padded edges) -- the method
SURVEY 8(d) names for bringing the 44.1 kHz fixture to 24 kHz -- with the filter designed here in float64 and the polyphase
dot products on the GPU (ryk_resample_poly).  Pinned against scipy.signal.resample_poly / firwin in tests/.
wav files: RIFF PCM 8/16/24/32-bit and IEEE float 32/64 are read; float32 is written (what librosa.output.write_wav did)."""
import math
import struct
from pathlib import Path
from typing import Optional, Tuple

import numpy

from .feature import Wave


def resample_filter(up: int, down: int) -> numpy.ndarray:
    """firwin(2 * 10 * max(up, down) + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up, float64."""
    max_rate = max(up, down)
    half_len = 10 * max_rate
    numtaps = 2 * half_len + 1
    cutoff = 1.0 / max_rate
    m = numpy.arange(numtaps, dtype=numpy.float64) - half_len
    h = cutoff * numpy.sinc(cutoff * m) * numpy.kaiser(numtaps, 5.0)
    h /= h.sum()
    return h * up


DRIFT_PHASES = 512          # clock drift stage (DESIGN.md §4l): phases of the prototype filter per input sample
DRIFT_HALF_WIDTH = 16       # ... and its half-width in input samples (zero crossings): 32 taps per output
DRIFT_BETA = 10.0           # ... and the Kaiser window's beta


def drift_filter(phases: int = DRIFT_PHASES, half_width: int = DRIFT_HALF_WIDTH, beta: float = DRIFT_BETA) -> numpy.ndarray:
    """The prototype filter of the clock drift stage (DESIGN.md DECIDE D3): a Kaiser-windowed sinc with its cutoff at Nyquist, sampled
    at `phases` points per input sample over [-half_width, half_width]: 2 * half_width * phases + 1 float64 values, entry k at
    t = k / phases - half_width.  The entries at integer t are exactly 0, except the centre, which is exactly 1, so a whole-sample
    position reads the input sample itself."""
    n = 2 * half_width * phases + 1
    t = numpy.arange(n, dtype=numpy.float64) / phases - half_width
    h = numpy.sinc(t) * numpy.i0(beta * numpy.sqrt(numpy.maximum(0.0, 1.0 - (t / half_width) ** 2))) / numpy.i0(beta)
    h[::phases] = 0.0
    h[half_width * phases] = 1.0
    return h


def resample_geometry(n_in: int, up: int, down: int) -> Tuple[int, int, int, int, int]:
    """(up, down) reduced by their gcd, n_out, n_pre_pad, n_pre_remove of scipy.signal.resample_poly."""
    g = math.gcd(up, down)
    up, down = up // g, down // g
    n_out = n_in * up
    n_out = n_out // down + bool(n_out % down)
    half_len = 10 * max(up, down)
    n_pre_pad = down - half_len % down
    n_pre_remove = (half_len + n_pre_pad) // down
    return up, down, n_out, n_pre_pad, n_pre_remove


def stream_input_geometry(rate: int, fs: int, buffer_time: float) -> Tuple[int, int, int]:
    """(n_in, n, delay) of a session at `fs` that takes its chunks at device rate `rate` (DESIGN.md DECIDE R1): n_in device samples per
    chunk, n model samples per step, and the delay in model samples -- the smallest for which every sample of step k's chunk,
    concat(zeros(delay), resample_poly(x))[k n:(k + 1) n], has its whole filter support inside the chunks received."""
    n_in, n = round(rate * buffer_time), round(fs * buffer_time)
    g = math.gcd(int(fs), int(rate))
    up, down = int(fs) // g, int(rate) // g
    if n_in * up != n * down:
        raise ValueError(f'a {buffer_time} s chunk at {rate} Hz is not a whole number of samples at {fs} Hz')
    return n_in, n, (10 * max(up, down)) // down


def stream_output_count(n_samples: int, rate: int, fs: int) -> int:
    """M: how many samples of resample_poly(y) (fs -> device rate `rate`) have their whole filter support inside the first
    `n_samples` samples of y -- what a session has returned once its synthesizer produced n_samples (DESIGN.md DECIDE R1)."""
    g = math.gcd(int(fs), int(rate))
    up, down = int(rate) // g, int(fs) // g
    return max(0, (n_samples * up - 1 - 10 * max(up, down)) // down + 1)


def resample(x: numpy.ndarray, rate_in: int, rate_out: int, engine=None) -> numpy.ndarray:
    """float32 signal at rate_in -> float32 signal at rate_out (ceil(len * rate_out / rate_in) samples)."""
    x = numpy.ascontiguousarray(x, dtype=numpy.float32)
    if rate_in == rate_out:
        return x.copy()
    from .engine import default_engine
    engine = engine or default_engine()
    g = math.gcd(int(rate_in), int(rate_out))
    up, down = int(rate_out) // g, int(rate_in) // g
    return engine.resample_poly(x, up, down, resample_filter(up, down))


def read_wav(path) -> Tuple[numpy.ndarray, int]:
    """-> (float32 mono samples in [-1, 1], sampling rate).  Multi-channel files are averaged (librosa.load(mono=True))."""
    data = Path(path).read_bytes()
    if data[:4] != b'RIFF' or data[8:12] != b'WAVE':
        raise ValueError(f'{path}: not a RIFF/WAVE file')
    pos, fmt, samples = 12, None, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack('<I', data[pos + 4:pos + 8])[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b'fmt ':
            tag, ch, rate, _, _, bits = struct.unpack('<HHIIHH', body[:16])
            if tag == 0xFFFE and size >= 26:                     # WAVE_FORMAT_EXTENSIBLE: the sub-format's first two bytes
                tag = struct.unpack('<H', body[24:26])[0]
            fmt = (tag, ch, rate, bits)
        elif cid == b'data':
            samples = body
        pos += 8 + size + (size & 1)
    if fmt is None or samples is None:
        raise ValueError(f'{path}: missing fmt / data chunk')
    tag, ch, rate, bits = fmt
    if tag == 1:
        if bits == 8:
            x = (numpy.frombuffer(samples, numpy.uint8).astype(numpy.float32) - 128.0) / 128.0
        elif bits == 16:
            x = numpy.frombuffer(samples, '<i2').astype(numpy.float32) / 32768.0
        elif bits == 24:
            b = numpy.frombuffer(samples, numpy.uint8).reshape(-1, 3).astype(numpy.int32)
            v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
            x = (v - ((v & 0x800000) << 1)).astype(numpy.float32) / 8388608.0
        elif bits == 32:
            x = (numpy.frombuffer(samples, '<i4').astype(numpy.float64) / 2147483648.0).astype(numpy.float32)
        else:
            raise ValueError(f'{path}: unsupported PCM width {bits}')
    elif tag == 3:
        x = numpy.frombuffer(samples, '<f4' if bits == 32 else '<f8').astype(numpy.float32)
    else:
        raise ValueError(f'{path}: unsupported wav format tag {tag}')
    if ch > 1:
        x = x[:len(x) // ch * ch].reshape(-1, ch).mean(axis=1).astype(numpy.float32)
    return x, int(rate)


def write_wav(path, wave: numpy.ndarray, sampling_rate: int) -> None:
    """IEEE float32 mono wav (librosa.output.write_wav's format for float input)."""
    x = numpy.ascontiguousarray(wave, dtype='<f4')
    body = x.tobytes()
    fmt = struct.pack('<HHIIHH', 3, 1, int(sampling_rate), int(sampling_rate) * 4, 4, 32)
    fact = struct.pack('<I', len(x))
    chunks = b'fmt ' + struct.pack('<I', len(fmt)) + fmt + b'fact' + struct.pack('<I', 4) + fact + b'data' + struct.pack('<I', len(body)) + body
    Path(path).write_bytes(b'RIFF' + struct.pack('<I', 4 + len(chunks)) + b'WAVE' + chunks)


def load_wave(path, sampling_rate: Optional[int] = None, engine=None) -> Wave:
    """librosa.load(path, sr=sampling_rate) as the reference uses it (check.py:80): mono float32, resampled on the GPU."""
    x, rate = read_wav(path)
    if sampling_rate is not None and sampling_rate != rate:
        x, rate = resample(x, rate, sampling_rate, engine), int(sampling_rate)
    return Wave(wave=x, sampling_rate=rate)


def save_wave(path, wave: Wave) -> None:
    write_wav(path, numpy.asarray(wave.wave, dtype=numpy.float32), wave.sampling_rate)
