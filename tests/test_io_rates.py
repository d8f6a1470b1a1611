"""Streaming resampling at a session's device rates (DESIGN.md DECIDE R1), on the CPU.

The geometry helpers of wave_io (chunk length n_in, input delay D, output count M_k) are checked against an independent numpy
transcription of the two streaming rules: a resampler that keeps only the samples it has been given, fed chunk by chunk, emitting a
sample as soon as its whole filter support has arrived.  Its concatenated output must be scipy.signal.resample_poly of the whole
signal (with the delay's leading zeros on the input side), and RealtimePipeline at the models' rate must not touch the new calls."""
import math

import numpy as np
import pytest
import scipy.signal as ss

from realtime_yukarin_b200 import synthetic, wave_io

FS = 24000
RATES = [16000, 32000, 44100, 48000, 96000]


def _ratio(r_from, r_to):
    g = math.gcd(r_from, r_to)
    return r_to // g, r_from // g


class _StreamingResampler:
    """Direct-form polyphase filter over the samples received so far.  Output i = sum_j x[j] h[half + i down - j up] is emitted once
    x[j_max(i)] has arrived (j_max(i) = floor((i down + half) / up)); samples before the signal are zero."""

    def __init__(self, up, down):
        self.up, self.down = up, down
        self.h = wave_io.resample_filter(up, down)
        self.half = (len(self.h) - 1) // 2
        self.x = np.zeros(0)
        self.emitted = 0

    def push(self, chunk, limit=None):
        self.x = np.concatenate([self.x, np.asarray(chunk, np.float64)])
        out = []
        while limit is None or len(out) < limit:
            c = self.half + self.emitted * self.down        # tap of x[0]
            jhi = c // self.up
            if jhi >= len(self.x):
                break
            jlo = max(0, -(-(c - len(self.h) + 1) // self.up))
            j = np.arange(jlo, jhi + 1)
            out.append(float(np.dot(self.x[jlo:jhi + 1], self.h[c - j * self.up])))
            self.emitted += 1
        return np.asarray(out)


@pytest.mark.parametrize('rate', RATES)
@pytest.mark.parametrize('T', [0.1, 0.3])
def test_input_geometry_matches_streaming_transcription(rate, T):
    """n_in, D: step k's model-rate chunk is concat(zeros(D), resample_poly(x))[k n:(k + 1) n] and D is the smallest delay for which
    the streaming resampler has every sample of that chunk after k + 1 chunks."""
    n_in, n, D = wave_io.stream_input_geometry(rate, FS, T)
    assert n_in == round(rate * T) and n == round(FS * T)
    up, down = _ratio(rate, FS)
    assert n_in * up == n * down
    K = 6
    x = np.random.default_rng(rate).standard_normal(K * n_in)
    rs = _StreamingResampler(up, down)
    have = []                                                             # model samples available after k + 1 chunks
    for k in range(K):
        rs.push(x[k * n_in:(k + 1) * n_in])
        have.append(rs.emitted)
    # smallest delay: every chunk's last sample (k + 1) n - D - 1 must be available
    d_min = max(max((k + 1) * n - have[k] for k in range(K)), 0)
    assert D == d_min, (rate, T, D, d_min)
    ref = ss.resample_poly(x, up, down, window=wave_io.resample_filter(up, down) / up)
    delayed = np.concatenate([np.zeros(D), ref])
    rs2 = _StreamingResampler(up, down)
    got = np.concatenate([np.zeros(D)] + [rs2.push(x[k * n_in:(k + 1) * n_in]) for k in range(K)])[:K * n]
    assert np.max(np.abs(got - delayed[:K * n])) <= 1e-12 * np.max(np.abs(x))


def test_input_chunk_must_be_whole():
    with pytest.raises(ValueError):
        wave_io.stream_input_geometry(44100, FS, 0.005)       # round(220.5) = 220 samples at 44.1 kHz are not 120 at 24 kHz
    # 0.1, 0.3 and 1.0 s are whole at every tabled rate
    for rate in (48000, 44100, 32000, 16000):
        for T in (0.1, 0.3, 1.0):
            wave_io.stream_input_geometry(rate, FS, T)


@pytest.mark.parametrize('rate', RATES)
def test_output_count_matches_streaming_transcription(rate):
    """M_k: the streaming resampler fed the synthesizer's samples in steps of random length (multiples of a block, some empty) emits
    exactly M_k samples in total after step k, and their concatenation is resample_poly(y)[:M_k]."""
    up, down = _ratio(FS, rate)
    rng = np.random.default_rng(rate)
    y = rng.standard_normal(40 * 1024)
    rs = _StreamingResampler(up, down)
    ref = ss.resample_poly(y, up, down, window=wave_io.resample_filter(up, down) / up)
    pos, outs = 0, []
    while pos < len(y):
        step = int(rng.integers(0, 5)) * 1024
        outs.append(rs.push(y[pos:pos + step]))
        pos += step
        M = wave_io.stream_output_count(min(pos, len(y)), rate, FS)
        assert rs.emitted == M, (rate, pos, rs.emitted, M)
    got = np.concatenate(outs)
    assert np.max(np.abs(got - ref[:len(got)])) <= 1e-12 * np.max(np.abs(y))


def test_pipeline_at_model_rate_uses_no_device_rate(small_models):
    """A 24 kHz config on the CPU stand-in never calls the device-rate entry points (the stand-in has none)."""
    from realtime_yukarin_b200.config import Config, VocodeMode
    from realtime_yukarin_b200.worker import RealtimePipeline
    from tests.fake_engine import OracleEngine

    class Strict(OracleEngine):
        def __getattr__(self, name):
            if name.startswith('session_set_') or name == 'session_io_geometry':
                raise AssertionError(f'{name} called at the model rate')
            raise AttributeError(name)

    fake = Strict(small_models['stage1_model_path'], small_models['stage2_model_path'])
    cfg = Config(input_device_name=None, output_device_name=None, input_rate=24000, output_rate=24000, frame_period=5.0, buffer_time=0.3,
                 extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                 output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0,
                 **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path', 'stage1_config_path',
                                                 'stage2_model_path', 'stage2_config_path')})
    pipe = RealtimePipeline(cfg, engine=fake, depth=1)
    x = synthetic.synthetic_speech(0.7, stream=2)
    out = pipe.process(x[:cfg.in_audio_chunk])
    assert len(out) == cfg.out_audio_chunk
    pipe.close()
