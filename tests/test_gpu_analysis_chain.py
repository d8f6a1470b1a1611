"""The session's front chain: cross-step buffer guards, D4C's coarse aperiodicity by selection, StoneMask's per-plan FFT bound.

  * Pipelining must not change a sample: at the headline configuration (0.3 s chunks, extras (0, 0.5, 0), base-64 models, FP16) the
    outputs of back-to-back device steps and of submit / collect with chunks in flight are bitwise equal to stepping one chunk at a
    time with a device synchronise in between, for a single session and for a 4-member group.  A guard that lets a step overwrite a
    buffer that an earlier step still reads shows up here as a difference.
  * D4C at 48 kHz (4096-point FFT, five coarse bands, all but the 65 largest of 2049 power values summed) against the oracle.
  * DIO contours that sit at f0_floor go through StoneMask plans whose shared memory is sized for f0_floor, and still match the oracle.
"""
import numpy as np
import pytest

from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import synthetic

pytestmark = pytest.mark.gpu

T, EXTRA, FS = 0.3, (0.0, 0.5, 0.0), 24000
N_CHUNKS = 68


def _load(engine, paths):
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=engine)
    SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=engine)


def _cfg():
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                         encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                         vocoder_buffer_size=1024)


def _chunks(members):
    n = round(T * FS)
    xs = [synthetic.synthetic_speech((N_CHUNKS + 1) * T, stream=90 + j) for j in range(members)]
    return [[np.ascontiguousarray(x[k * n:(k + 1) * n]) for x in xs] for k in range(N_CHUNKS)]      # [step][member]


def _run_device(engine, chunks, sync_each):
    """Every step's output of fresh sessions (grouped when there are several), steps pushed from device memory with one output slot
    per step; sync_each: a device synchronise after every step, else all steps back to back."""
    import torch
    B = len(chunks[0])
    sids = [engine.session_create(_cfg()) for _ in range(B)]
    gid = engine.group_create(sids) if B > 1 else None
    n, cap = len(chunks[0][0]), engine.session_io_geometry(sids[0])['max_out']
    d_in = torch.from_numpy(np.stack([np.stack(c) for c in chunks])).cuda()
    d_out = torch.full((N_CHUNKS, B, cap), np.nan, dtype=torch.float64, device='cuda')
    d_n = torch.zeros((N_CHUNKS, B), dtype=torch.int32, device='cuda')
    engine.synchronize()
    for k in range(N_CHUNKS):
        if gid is None:
            engine.session_push_device(sids[0], d_in[k, 0].data_ptr(), n, d_out[k, 0].data_ptr(), cap, d_n[k, 0:].data_ptr())
        else:
            engine.group_push_device(gid, [d_in[k, j].data_ptr() for j in range(B)], n, [d_out[k, j].data_ptr() for j in range(B)], cap,
                                     [d_n[k, j:].data_ptr() for j in range(B)])
        if sync_each:
            engine.synchronize()
    engine.synchronize()
    torch.cuda.synchronize()
    outs, ns = d_out.cpu().numpy(), d_n.cpu().numpy()
    if gid is not None:
        engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    return [[outs[k, j, :ns[k, j]].copy() for j in range(B)] for k in range(N_CHUNKS)]


def _run_submit(engine, chunks, depth):
    """Every step's output through the host API with `depth` steps in flight."""
    B = len(chunks[0])
    sids = [engine.session_create(_cfg()) for _ in range(B)]
    gid = engine.group_create(sids) if B > 1 else None
    cap = engine.session_io_geometry(sids[0])['max_out']
    bufs = [[np.empty(cap) for _ in range(B)] for _ in range(8)]
    tickets, outs = [], []

    def collect():
        t = tickets.pop(0)
        if gid is None:
            outs.append([engine.session_collect(sids[0], t, bufs[t % 8][0]).copy()])
        else:
            outs.append([o.copy() for o in engine.group_collect(gid, t, bufs[t % 8])])
    for k in range(N_CHUNKS):
        tickets.append(engine.session_submit(sids[0], chunks[k][0]) if gid is None else engine.group_submit(gid, chunks[k]))
        if len(tickets) > depth:
            collect()
    while tickets:
        collect()
    if gid is not None:
        engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    return outs


@pytest.mark.parametrize('members', [1, 4])
def test_pipelined_steps_bitwise_equal_stepwise(engine, full_models, members):
    _load(engine, full_models)
    engine.set_precision('fp16')
    chunks = _chunks(members)
    ref = _run_device(engine, chunks, sync_each=True)
    produced = sum(len(o) for step in ref for o in step)
    assert produced > N_CHUNKS * members * 4096, produced          # the comparison covers real output, not empty steps
    runs = {'back-to-back device steps': _run_device(engine, chunks, sync_each=False),
            'submit / collect, 4 in flight': _run_submit(engine, chunks, 4),
            'submit / collect, 5 in flight': _run_submit(engine, chunks, 5)}
    for name, got in runs.items():
        for k in range(N_CHUNKS):
            for j in range(members):
                a, b = got[k][j], ref[k][j]
                assert len(a) == len(b), (name, k, j, len(a), len(b))
                assert np.array_equal(a, b), (name, k, j, float(np.max(np.abs(a - b))) if len(a) else 0.0)


def test_world_analysis_matches_oracle_48k(engine):
    """D4C at 48 kHz: fft 4096, 2049 bins, nap = 5, boundary 64 (the 65 largest power values left out of each band's sum)."""
    cfg = opipe.PathConfig(fs=48000, fft_length=2048)
    for stream, seconds in ((6, 0.6), (7, 0.3)):
        x = synthetic.synthetic_speech(seconds, stream=stream, fs=cfg.fs)
        ref = opipe.extract_features(x, cfg)
        got = engine.world_analyze(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length, cfg.order, cfg.alpha)
        f0r, f0g = ref['f0'].ravel(), got['f0']
        assert np.array_equal(f0r != 0, f0g != 0), (f0r, f0g)
        assert np.allclose(f0g, f0r, rtol=1e-6, atol=0)
        assert np.array_equal(ref['voiced'].ravel(), got['voiced'])
        assert ref['voiced'].sum() > 0
        assert np.allclose(np.log(got['sp']), np.log(ref['sp']), atol=2e-4), np.abs(np.log(got['sp']) - np.log(ref['sp'])).max()
        assert np.allclose(got['ap'], ref['ap'], rtol=1e-4, atol=1e-6), np.abs(got['ap'] - ref['ap']).max()
        assert np.allclose(got['mc'], ref['mc'], atol=2e-4), np.abs(got['mc'] - ref['mc']).max()


def _glide(f_lo, f_hi, seconds=1.0, seed=0):
    """A harmonic tone gliding from f_lo to f_hi Hz at 24 kHz, with a little noise."""
    n = int(seconds * FS)
    ph = 2 * np.pi * np.cumsum(np.linspace(f_lo, f_hi, n)) / FS
    x = sum(np.sin(k * ph) / k for k in range(1, 12)) * 0.2
    return (x + np.random.default_rng(seed).normal(0, 1e-3, n)).astype(np.float32)


@pytest.mark.parametrize('f0_floor, glide', [(71.0, (70.0, 80.0)), (150.0, (148.0, 170.0))])
def test_stonemask_at_f0_floor_matches_oracle(engine, f0_floor, glide):
    """f0_floor 71 Hz bounds StoneMask's FFT at 2048 points at 24 kHz, 150 Hz at 1024: the frames whose f0 sits at the floor use the
    largest FFT such a plan holds.  DIO + StoneMask must still equal the oracle's (which sizes every frame's FFT on its own) to 1e-9."""
    x = _glide(*glide)
    f0_dio, t = oworld.dio(x.astype(np.float64), FS, 5.0, f0_floor, 800.0)
    f0_ref = oworld.stonemask(x.astype(np.float64), FS, t, f0_dio)
    voiced = f0_dio[f0_dio > 0]
    assert len(voiced) > 100 and voiced.min() < f0_floor * 1.01, voiced.min()      # the contour reaches the floor
    f0, _ = engine.world_f0(x, FS, 5.0, f0_floor, 800.0)
    assert np.array_equal(f0 != 0, f0_ref != 0)
    assert np.allclose(f0, f0_ref, rtol=1e-9, atol=0), np.abs(f0 - f0_ref).max()
