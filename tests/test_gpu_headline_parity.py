"""GPU parity AT THE BENCHMARKED CONFIGURATION: full-width models (base 64), FP16 operands on wgmma, the pipelined session
(`ryk_session_submit / collect`, `ryk_group_submit / collect`) -- the exact path `bench.py` times -- against the CPU oracle stream.

BASELINE.json configs covered: [1] single stream 0.3 s, extras (0,0.5,0) (Tw 260 -> Tp 384); [2] the buffer sweep 0.1 / 0.3 / 1.0 s
incl. the `pad == 0` branch of convert_stream.py:40-42 (extras (0,0,0)); [4] the 8-per-GPU grouped shape (Tp 512, batch 8).
Reference behaviour matched: check.py:118-127 (chunk loop), yukarin_wrapper/voice_changer.py:24-42 (convert).

Tolerances (north_star: "per-frame spectral L2 and sample RMSE", target 1e-3 sample RMSE):
  * waveform: sample RMSE <= 1e-3 absolute (signal RMS ~0.1), asserted per configuration and per group member;
  * waveform spectra: per-frame log-magnitude STFT distance (frames above -60 dB), RMS over bins <= 0.1 (about 0.9 dB), asserted;
  * converted spectral envelope (the stage-2 output the synthesizer consumes): per-frame log-spectrum L2 / sqrt(bins) <= 1e-2,
    max <= 6e-2, asserted at Tp = 384 / 512 / 640 and on a full convert window at the headline shape.
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()


def _load(engine, paths):
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    ac = AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=engine)
    sr = SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=engine)
    return ac, sr, f0c


def _session_cfg(T, extra):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=24000, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                         buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                         threshold_db=60.0, vocoder_buffer_size=1024)


def _rmse(a, b):
    return float(np.sqrt(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2)))


def _stft_logmag(y, n_fft=1024, hop=256):
    y = np.asarray(y, np.float64)
    if len(y) < n_fft:
        return np.zeros((0, n_fft // 2 + 1))
    w = np.hanning(n_fft)
    n = 1 + (len(y) - n_fft) // hop
    fr = np.stack([y[i * hop:i * hop + n_fft] * w for i in range(n)])
    return np.abs(np.fft.rfft(fr, axis=1))


def _waveform_spectral_distance(y, r):
    """per-frame RMS (over bins) of the log-magnitude difference, over frames / bins above -60 dB of the reference peak"""
    Y, R = _stft_logmag(y), _stft_logmag(r)
    if len(R) == 0:
        return 0.0
    floor = R.max() * 1e-3
    keep = R.max(axis=1) > floor * 10
    if not keep.any():
        return 0.0
    d = np.log(np.maximum(Y[keep], floor)) - np.log(np.maximum(R[keep], floor))
    return float(np.sqrt((d ** 2).mean(axis=1)).max())


def _logspec_err(a, b):
    d = np.log(a.astype(np.float64)) - np.log(b.astype(np.float64))
    return float(np.sqrt((d ** 2).mean(axis=1)).max()), float(np.abs(d).max())


HEADLINE = [
    # buffer_time, extras, chunks   (Tw -> Tp)
    (0.3, (0.0, 0.5, 0.0), 12),     # BASELINE config 2: 260 -> 384  (what bench.py times)
    (0.1, (0.0, 0.5, 0.0), 12),     # config 3: 220 -> 256
    (1.0, (0.0, 0.5, 0.0), 6),      # config 3 / config.yaml: 400 -> 512
    (0.3, (0.0, 0.0, 0.0), 12),     # config 3, no overlap: the pad == 0 branch (60 -> 128)
    (0.3, (0.1, 0.5, 0.1), 10),     # all three overlaps
]


@pytest.mark.parametrize('T,extra,nchunks', HEADLINE)
def test_fp16_full_model_session_matches_oracle(engine, full_models, T, extra, nchunks):
    """>= 10 chunks (6 one-second chunks) through ryk_session_submit / collect, 3 in flight, FP16 tensor-core mode, base-64 models."""
    ac, sr, f0c = _load(engine, full_models)
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    engine.set_precision('fp16')
    sid = engine.session_create(_session_cfg(T, extra))
    orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
    n = round(T * 24000)
    x = synthetic.synthetic_speech((nchunks + 1) * T, stream=91)
    buf = np.empty(65536)
    tickets, outs = [], []
    for k in range(nchunks):
        tickets.append(engine.session_submit(sid, x[k * n:(k + 1) * n]))
        if len(tickets) > 3:
            outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    while tickets:
        outs.append(engine.session_collect(sid, tickets.pop(0), buf).copy())
    refs = [orc.push(x[k * n:(k + 1) * n]) for k in range(nchunks)]
    engine.session_destroy(sid)
    assert [len(o) for o in outs] == [len(r) for r in refs]
    y, r = np.concatenate(outs), np.concatenate(refs)
    assert len(y) > 0
    rmse, rms = _rmse(y, r), float(np.sqrt(np.mean(r ** 2)))
    lsd = _waveform_spectral_distance(y, r)
    print(f'HEADLINE fp16 base-64 session T={T} extra={extra}: {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), '
          f'per-frame log-STFT distance {lsd:.3e}')
    assert rms > 1e-2                      # the stream is not silent
    assert rmse <= 1e-3, rmse
    assert lsd <= 0.1, lsd


def test_fp16_full_model_group_of_8_matches_oracle_streams(engine, full_models):
    """BASELINE config 5 shape: 8 streams per GPU, 1.0 s chunks (Tp 512), ONE batched stage-2 forward per step (ryk_group_*)."""
    ac, sr, f0c = _load(engine, full_models)
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    engine.set_precision('fp16')
    T, extra, B, nchunks = 1.0, (0.0, 0.5, 0.0), 8, 4
    n = round(T * 24000)
    xs = [synthetic.synthetic_speech((nchunks + 1) * T, stream=120 + i) for i in range(B)]
    sids = [engine.session_create(_session_cfg(T, extra)) for _ in range(B)]
    gid = engine.group_create(sids)
    bufs = [[np.empty(65536) for _ in range(B)] for _ in range(8)]
    tickets, outs = [], [[] for _ in range(B)]

    def collect():
        t = tickets.pop(0)
        for i, o in enumerate(engine.group_collect(gid, t, bufs[t % 8])):
            outs[i].append(o.copy())
    for k in range(nchunks):
        tickets.append(engine.group_submit(gid, [x[k * n:(k + 1) * n] for x in xs]))
        if len(tickets) > 2:
            collect()
    while tickets:
        collect()
    engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    worst = 0.0
    for i in range(B):
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
        refs = [orc.push(xs[i][k * n:(k + 1) * n]) for k in range(nchunks)]
        assert [len(o) for o in outs[i]] == [len(r) for r in refs], i
        y, r = np.concatenate(outs[i]), np.concatenate(refs)
        rmse = _rmse(y, r)
        worst = max(worst, rmse)
        print(f'HEADLINE fp16 base-64 group of 8, member {i}: {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {float(np.sqrt(np.mean(r ** 2))):.3e})')
        assert rmse <= 1e-3, (i, rmse)
    print(f'HEADLINE group of 8 worst member RMSE {worst:.3e}')


@pytest.mark.parametrize('T', [260, 400, 600])
def test_fp16_full_width_stage2_alone(engine, full_models, T):
    """Stage 2 alone at the production heights (Tp = 384 / 512 / 640 x 512 bins, base 64) vs oracle stage2_convert."""
    ac, sr, f0c = _load(engine, full_models)
    p2 = onets.load_npz(full_models['stage2_model_path'])
    rng = np.random.default_rng(T)
    sp = np.exp(-9 + 2.5 * rng.standard_normal((T, 513))).astype(np.float32)
    ref = onets.stage2_convert(sp, p2, backend='torch')
    engine.set_precision('fp16')
    got = engine.stage2_convert(sp)
    l2, mx = _logspec_err(got, ref)
    print(f'HEADLINE stage 2 alone T={T}: fp16-tc per-frame log-L2 {l2:.2e}, max {mx:.2e}')
    assert l2 <= 1e-2 and mx <= 6e-2, (l2, mx)


def test_fp16_full_model_convert_window_spectra(engine, full_models):
    """One full convert window at the headline shape (Tw 260) through ryk_convert_window: the converted spectral envelope the
    synthesizer consumes, per frame, vs the oracle (gate decisions / f0 / ap exact)."""
    ac, sr, f0c = _load(engine, full_models)
    p1, p2 = onets.load_npz(full_models['stage1_model_path']), onets.load_npz(full_models['stage2_model_path'])
    x = synthetic.synthetic_speech(1.3, stream=17)
    enc = opipe.extract_features(x, CFG)
    ref = opipe.convert_window(x, enc, CFG, p1, p2, f0c.stats(), backend='torch')
    engine.set_precision('fp16')
    out = engine.convert_window(x, CFG.fs, CFG.fft_length, CFG.hop, 60.0, enc['f0'].ravel(), enc['ap'], enc['mc'], enc['voiced'].ravel(),
                                CFG.order, CFG.alpha, CFG.fft_length)
    assert np.array_equal(np.asarray(out['voiced']).ravel().astype(bool), ref['voiced'].ravel())
    assert np.allclose(np.asarray(out['f0']).ravel(), ref['f0'].ravel(), rtol=1e-6)
    l2, mx = _logspec_err(out['sp'], ref['sp'])
    print(f'HEADLINE convert window Tw=260 fp16 base-64: per-frame log-L2 {l2:.2e}, max {mx:.2e}')
    assert l2 <= 1e-2 and mx <= 6e-2, (l2, mx)


def test_soak_1200_chunks_ring_wraps(engine, small_models):
    """One session, 1200 consecutive 0.3 s chunks (6 minutes of audio) through submit / collect with 3 in flight, compared with the
    oracle stream chunk by chunk: crosses the synthesizer's noise-ring refills (every 2^21 samples = 87 s), wraps the pulse ring
    (2^15 pulses) and the 8-slot event / staging rings 150 times (VERDICT r1 item 8)."""
    ac, sr, f0c = _load(engine, small_models)
    p1, p2 = onets.load_npz(small_models['stage1_model_path']), onets.load_npz(small_models['stage2_model_path'])
    engine.set_precision('fp16')
    T, extra, nchunks = 0.3, (0.0, 0.5, 0.0), 1200
    sid = engine.session_create(_session_cfg(T, extra))
    orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=extra, backend='torch')
    n = round(T * 24000)
    base = synthetic.synthetic_speech(30.0, stream=55)          # 100 chunks of audio, cycled
    per = len(base) // n
    buf = np.empty(65536)
    tickets, worst, total_sq, total_n, sig_sq = [], 0.0, 0.0, 0, 0.0

    def check(k_out, y):
        nonlocal worst, total_sq, total_n, sig_sq
        r = orc.push(base[(k_out % per) * n:(k_out % per + 1) * n])
        assert len(y) == len(r), (k_out, len(y), len(r))
        if len(r):
            e = float(np.sqrt(np.mean((y - r) ** 2)))
            worst = max(worst, e)
            total_sq += float(np.sum((y - r) ** 2)); total_n += len(r); sig_sq += float(np.sum(r ** 2))
            assert e <= 2e-3, (k_out, e)                       # per chunk; the whole-run RMSE is asserted below
    k_out = 0
    for k in range(nchunks):
        tickets.append(engine.session_submit(sid, base[(k % per) * n:(k % per + 1) * n]))
        if len(tickets) > 3:
            check(k_out, engine.session_collect(sid, tickets.pop(0), buf).copy()); k_out += 1
    while tickets:
        check(k_out, engine.session_collect(sid, tickets.pop(0), buf).copy()); k_out += 1
    engine.session_destroy(sid)
    rmse, rms = (total_sq / total_n) ** 0.5, (sig_sq / total_n) ** 0.5
    print(f'SOAK {nchunks} chunks ({nchunks * T:.0f} s of audio, {total_n} samples): sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), worst chunk {worst:.3e}')
    assert rmse <= 1e-3
