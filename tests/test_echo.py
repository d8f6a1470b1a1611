"""The FP64 reference of the echo canceller (DESIGN.md DECIDE E1-E4) and RealtimePipeline's far end, without a GPU:

  * fed in chunks with its state carried it is exactly the whole-signal canceller, whatever the chunk length;
  * with the far end alone through a synthetic room it converges to a stated echo return loss enhancement;
  * during double talk the two-path control keeps the near-end voice better than a single NLMS filter;
  * it reconverges after the echo path changes, and a bulk delay covers an echo the taps alone cannot reach;
  * RealtimePipeline pairs each input chunk with the played stream, also when the output chunks are longer or shorter.

The far end is the golden speech looped; the rooms are tests/echo_oracle.room_ir (bulk delay, 100 ms exponential tail, gain 0.5).
"""
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic, wave_io

from . import denoise_oracle as DO
from . import echo_oracle as E
from .fake_engine import OracleEngine

FS = 24000
GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'


def _far(seconds):
    x, fs = wave_io.read_wav(GOLDEN)
    assert fs == FS
    return np.tile(np.asarray(x, np.float32), int(np.ceil(seconds * FS / len(x))))[:round(seconds * FS)]


def _residual_db(z, echo, a, b):
    """how far the residual z lies under the echo over [a, b) seconds, in dB"""
    s = slice(round(a * FS), round(b * FS))
    return -E.level_db(z[s], echo[s])


@pytest.mark.parametrize('chunk', [7200, 1337, 127])
def test_chunks_with_carried_state_are_the_whole_signal(chunk):
    far = _far(1.5)
    mic = (E.echo_of(far, E.room_ir(30)) + 0.3 * synthetic.synthetic_speech(1.5, stream=5)).astype(np.float32)
    phi = DO.frame_powers(mic, 3, 40).mean(axis=0)
    for kw in (dict(), dict(suppression_db=12.0, phi=phi, delay_frames=3, taps=7)):
        whole = E.echo_cancel(mic, far, **kw)
        o = E.EchoOracle(**{k: v for k, v in kw.items()})
        pad = np.zeros(DO.D, np.float32)
        m, f = np.concatenate([mic, pad]), np.concatenate([far, pad])
        got = np.concatenate([o.push(m[a:a + chunk], f[a:a + chunk]) for a in range(0, len(m), chunk)])[DO.D:]
        assert np.array_equal(got, whole), kw


def test_far_end_alone_converges():
    # measured on this oracle: 27.3 dB (30 ms) and 17.7 dB (120 ms, where 32 taps = 171 ms cut the 100 ms tail short) over 4-6 s
    far = _far(6.0)
    for delay_ms, floor in ((30, 23.0), (120, 15.0)):
        echo = E.echo_of(far, E.room_ir(delay_ms)).astype(np.float32)
        z, o = E.echo_cancel(echo, far, 32, 0, oracle=True)
        got = _residual_db(z, echo, 4.0, 6.0)
        print(f'far end alone, {delay_ms} ms room: residual {got:.1f} dB under the echo over 4-6 s')
        assert got >= floor, (delay_ms, got)
    assert o.copies.sum() > 0


def test_double_talk_keeps_the_near_end_and_beats_a_single_filter():
    # 2 s of far end alone, then 4 s of double talk with the near-end voice 6 dB under the echo.  Measured on this oracle: the residual
    # echo lies 13.7 dB under the echo with the two-path control and 10.2 dB with the single filter.
    far = _far(6.0)
    echo = E.echo_of(far, E.room_ir(30))
    near = synthetic.synthetic_speech(4.0, stream=3)
    near = near / np.sqrt(np.mean(near ** 2)) * np.sqrt(np.mean(echo ** 2)) * 10 ** (-6 / 20)
    t0 = 2 * FS
    mic = echo.copy()
    mic[t0:] += near[:len(mic) - t0]
    mic = mic.astype(np.float32)
    res = {}
    for two_path in (True, False):
        z = E.echo_cancel(mic, far, 32, 0, two_path=two_path).astype(np.float64)
        res[two_path] = -E.level_db(z[t0:] - near[:len(z) - t0], echo[t0:])
        print(f'double talk, {"two-path" if two_path else "single filter"}: residual echo {res[two_path]:.1f} dB under the echo')
    assert res[True] >= 11.0 and res[True] >= res[False] + 2.0, res


def test_reconverges_after_the_echo_path_changes():
    # the room changes at 3 s (another tail, 30 -> 60 ms delay).  Measured on this oracle: 25.6 dB before, 3.7 dB in the first
    # 0.25 s after, 18.7 dB from 1.5 s to 3 s after the change
    far = _far(6.0)
    e1, e2 = E.echo_of(far, E.room_ir(30, seed=1)), E.echo_of(far, E.room_ir(60, seed=2))
    mic = np.where(np.arange(len(far)) < 3 * FS, e1, e2).astype(np.float32)
    z = E.echo_cancel(mic, far, 32, 0)
    before, just_after, later = _residual_db(z, mic, 2.0, 3.0), _residual_db(z, mic, 3.0, 3.25), _residual_db(z, mic, 4.5, 6.0)
    print(f'echo path change at 3 s: {before:.1f} dB before, {just_after:.1f} dB right after, {later:.1f} dB 1.5-3 s after')
    assert before >= 22.0 and just_after < 10.0 and later >= 15.0


def test_a_bulk_delay_reaches_an_echo_the_taps_alone_cannot():
    # an echo at 150 ms: 16 taps after 26 frames (139 ms) cover it; 16 taps alone reach 85 ms.  Measured: 23.6 dB and 3.2 dB.
    far = _far(6.0)
    echo = E.echo_of(far, E.room_ir(150, seed=3)).astype(np.float32)
    covered = _residual_db(E.echo_cancel(echo, far, 16, 26), echo, 3.0, 6.0)
    short = _residual_db(E.echo_cancel(echo, far, 16, 0), echo, 3.0, 6.0)
    print(f'150 ms echo: {covered:.1f} dB with delay_frames = 26, {short:.1f} dB without')
    assert covered >= 20.0 and short < 5.0


def test_suppression_zero_is_the_linear_canceller_and_more_suppresses_more():
    far = _far(2.0)
    echo = E.echo_of(far, E.room_ir(30)).astype(np.float32)
    lin = E.echo_cancel(echo, far)
    assert np.array_equal(E.echo_cancel(echo, far, suppression_db=0.0), lin)
    assert _residual_db(E.echo_cancel(echo, far, suppression_db=20.0), echo, 1.0, 2.0) > _residual_db(lin, echo, 1.0, 2.0) + 1.0


# ---- RealtimePipeline's far end over the oracle-backed stand-in ----
class EchoEngine(OracleEngine):
    """OracleEngine with the session's echo canceller in front of StreamOracle; it records the far end each submitted chunk got."""

    def session_echo_cancel(self, sid, taps=32, delay_ms=0.0):
        S = self.sessions[sid]
        S['echo'] = E.EchoOracle(taps, round(delay_ms * FS / 1000 / DO.H))
        S['far'], S['refs'] = None, []

    def session_set_echo_suppression(self, sid, db):
        self.sessions[sid]['echo'].set_suppression(db)

    def session_echo_reference(self, sid, far):
        self.sessions[sid]['far'] = np.array(far, np.float32)

    def session_submit(self, sid, wave):
        S = self.sessions[sid]
        if 'echo' in S:
            far = S['far'] if S['far'] is not None else np.zeros(len(wave), np.float32)
            assert len(far) == len(wave)
            S['refs'].append(far)
            S['far'] = None
            wave = S['echo'].push(wave, far)
        return super().session_submit(sid, wave)


def _config(small_models, **kw):
    from realtime_yukarin_b200.config import Config, VocodeMode
    fields = dict(input_device_name=None, output_device_name=None, input_rate=FS, output_rate=FS, frame_period=5.0, buffer_time=0.1,
                  extract_f0_mode=VocodeMode.WORLD, vocoder_buffer_size=1024, input_scale=1.0, output_scale=1.0, input_silent_threshold=60.0,
                  output_silent_threshold=80.0, encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0)
    fields.update(kw)
    return Config(**fields, **{k: small_models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                           'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})


def _out_chunk(base, n):
    """a Config whose output chunks are n samples: unequal chunk sizes at one rate, as a card with its own buffer size gives them"""
    class C(type(base)):
        @property
        def out_audio_chunk(self):
            return n
    return C(**{k: getattr(base, k) for k in base.__dataclass_fields__})


@pytest.mark.parametrize('out_ratio', [1.0, 0.75, 1.5])
def test_the_pipeline_pairs_each_chunk_with_the_played_stream(small_models, out_ratio):
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models)
    n_in = cfg.in_audio_chunk
    cfg = _out_chunk(cfg, round(out_ratio * n_in))
    fake = EchoEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    steps = 14
    x = synthetic.synthetic_speech((steps + 1) * 0.1, stream=29, silence_fraction=0.0)
    pipe = RealtimePipeline(cfg, engine=fake, echo_cancel=True, echo_taps=8, echo_suppression=6.0)
    played = []
    try:
        for k in range(steps):
            played.append(pipe.process(x[k * n_in:(k + 1) * n_in], block=True))
    finally:
        refs = fake.sessions[pipe._sid]['refs']
        pipe.close()
    assert all(len(p) == cfg.out_audio_chunk for p in played)
    assert any(np.any(p != 0) for p in played), 'the stand-in played nothing: the check below would be empty'
    # chunk i's far end: the next n_in samples of the played stream after n_in zeros, silence where it ran short
    fifo = np.zeros(n_in, np.float32)
    for i, r in enumerate(refs):
        want = np.concatenate([fifo[:n_in], np.zeros(max(0, n_in - len(fifo)), np.float32)])
        assert np.array_equal(r, want), i
        fifo = np.concatenate([fifo[n_in:], played[i]])
    if out_ratio == 1.0:
        assert all(np.array_equal(refs[i], played[i - 1]) for i in range(1, steps))


def test_a_closed_loop_never_amplifies_and_converges_when_the_speaker_stops(small_models):
    # The far end of a voice changer is its own converted input.  While the speaker talks, the background filter can learn to predict
    # the voice from the far end and pass the copy test; the foreground filter is cleared whenever it makes the output louder than the
    # microphone (E3).  Measured on this loop: every chunk at -0.0 dB or above, 19.5-20.9 dB over the last 10 chunks (without the
    # clear: -4 to -9 dB while talking and -21 to -29 dB after)
    from realtime_yukarin_b200.worker import RealtimePipeline
    cfg = _config(small_models, buffer_time=0.3)
    fake = EchoEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    n, steps, talk = cfg.in_audio_chunk, 30, 15
    near = synthetic.synthetic_speech((steps + 1) * 0.3, stream=861).astype(np.float32)
    near[talk * n:] = 0.0
    ir = E.room_ir(30, seed=861)
    pipe = RealtimePipeline(cfg, engine=fake, echo_cancel=True)
    played, erle = [np.zeros(n, np.float32)], []
    try:
        for k in range(steps):
            echo = E.echo_of(np.concatenate(played), ir)[k * n:(k + 1) * n]
            played.append(pipe.process((near[k * n:(k + 1) * n] + echo).astype(np.float32), block=True))
            erle.append(fake.sessions[pipe._sid]['echo'].erle_db())
    finally:
        pipe.close()
    print(f'closed loop on the oracle: ERLE per chunk {[round(float(e), 1) for e in erle]}')
    assert min(erle[2:]) >= -0.5 and float(np.mean(erle[-10:])) >= 17.0


def test_the_pipeline_refuses_echo_cancel_at_unequal_rates(small_models):
    from realtime_yukarin_b200.worker import RealtimePipeline
    fake = EchoEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    with pytest.raises(ValueError):
        RealtimePipeline(_config(small_models, output_rate=48000), engine=fake, echo_cancel=True)
    assert not getattr(fake, 'sessions', None)
