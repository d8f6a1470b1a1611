"""The FP16 stage-2 U-Net (conv_tc.cu wgmma layers, conv_direct.cu edge layers) against the oracle's forward at every window height a
session can run it with, at batch sizes a session group stacks, and at the largest group at the largest window.

Elsewhere the whole forward meets the oracle only at Tp 128 / 384 / 512 / 640 and the batch-8 headline group; the banded and tail-skipped
forwards of the other heights are compared with the device's own full forward, and the session geometries reach the oracle only
through the synthesized waveform.  Here the stage-2 output itself is compared with oracle.nets.unet_forward on the same input:

* the full forward at every height of tests/session_geometry.py (Tp 128, 256, 512, 1024, 1408, 1920), and at Tp 768 and 1280;
* batches of 3, 5 and 8 members with different data at Tp 768, 1280 and 1920, each member against its own oracle forward.  The bottleneck
  layers' split-K factor depends on the batch's tile count; the split of layer c5 is asserted per case, so that the cases keep covering
  both a split and an unsplit c5 if the planner changes.  (Batch 8 at Tp 1280 is left out: on an H100 SXM its layers c5 .. d2 run at
  the split-K factors of batch 8 at Tp 1920);
* a group of 64 members at Tp 1920, whose 64-channel full-resolution activations (c0's output, d6's output) hold 64 * 1920 * 512 * 64
  = 4.0e9 elements, past 2^31;
* the banded (mode 1) and tail-skipped (mode 3) kept rows of each height, against the oracle rather than the device's full forward;
* engine.stage2_convert (column-minimum padding, U-Net, edge-padded epilogue) at T = Tw of the Tp 1024 and 1920 session windows.

Inputs are log-spectra of the test_gpu_stage2_tail._padded_input construction (rows >= Tw repeat the column minimum, as a session pads its
window), rounded to FP16-representable values.  Tolerance: the stage-2 one of test_gpu_stage2_band._check_kept and
test_gpu_headline_parity, per-frame log-domain RMS <= 1e-2 and max <= 6e-2.  The oracle runs in float32 on torch's CPU convolutions: a
float64 forward at Tp 1920 takes minutes, and float32 accumulation-order noise (~1e-5, see test_gpu_conv_layers._ref32) is three orders
below the bound.  A member's input is seeded by (Tp, member), and its oracle output is cached, so the full, batched and banded cases of
one height share them.
"""
import functools

import numpy as np
import pytest

from oracle import nets as onets
from realtime_yukarin_b200 import engine as eng

from .session_geometry import BY_ID, GEOMETRIES, Geometry, stage2_cases
from .test_gpu_stage2_band import W, _load_stage2
from .test_gpu_stage2_tail import _padded_input

RMS_TOL, MAX_TOL = 1e-2, 6e-2

# session windows at the heights the batched cases add, and one at Tp 1920 with more than G9's single padding row, so that the
# tail-skipped case there skips rows
EXTRA_GEOMETRIES = [
    Geometry('S768', 0.5, (0.0, 1.5, 0.0)),         # Tw 700
    Geometry('S1280', 1.0, (0.0, 2.5, 0.0)),        # Tw 1200
    Geometry('S1920', 1.0, (0.0, 4.0, 0.0)),        # Tw 1800
]


def _heights():
    """Tp -> the session window of that height with the most padding rows"""
    by_tp = {}
    for g in GEOMETRIES + EXTRA_GEOMETRIES:
        if g.Tp not in by_tp or g.Tw < by_tp[g.Tp].Tw:
            by_tp[g.Tp] = g
    return dict(sorted(by_tp.items()))


HEIGHTS = _heights()                                   # Tp 128, 256, 512, 768, 1024, 1280, 1408, 1920

# (Tp, B, whether layer c5 splits K): c5 has B * ceil(Tp / 256) * 4 output tiles, and the planner splits K when a layer has fewer tiles
# than two per SM (264 on an H100 SXM)
BATCHED = [(768, 3, True), (768, 5, True), (768, 8, True),
           (1280, 3, True), (1280, 5, True),
           (1920, 3, True), (1920, 5, False), (1920, 8, False)]
# the k4 layers whose split-K factor these batches change: c5 .. c7, d0 .. d2 (layer indices of the U-Net)
SPLIT_LAYERS = (5, 6, 7, 8, 9, 10)

# the largest group (csrc/conv.h kMaxGroupBatch) at the largest window; every member is compared with its own batch-of-one forward, and
# these members with the oracle
BIG_TP, BIG_B = 1920, 64
BIG_SEED = 2031


def _seed(Tp, member):
    return Tp * 1000 + member


def _member_input(Tp, member):
    """[Tp][W] network input of one member: rows >= Tw hold the column minimum, every value FP16-representable"""
    Tw = HEIGHTS[Tp].Tw
    x = _padded_input(1, Tp, Tw, _seed(Tp, member))[0]
    return x.astype(np.float16).astype(np.float32)     # monotone rounding: the padded rows still hold the column minimum


@functools.lru_cache(maxsize=None)
def _params(path):
    return onets.load_npz(path)


@functools.lru_cache(maxsize=None)
def _oracle_cached(path, Tp, member):
    return onets.unet_forward(_member_input(Tp, member)[None], _params(path), ndim=2, backend='torch')[0]


def _oracle(models, Tp, member):
    """float32 CPU forward of the member's input, [Tp][W]"""
    return _oracle_cached(str(models['stage2_model_path']), Tp, member)


def _errors(got, ref):
    """(worst per-frame RMS, max |difference|, rows over the tolerance) of two [rows][W] log-spectra"""
    d = got.astype(np.float64) - ref
    row_rms = np.sqrt((d ** 2).mean(axis=1))
    row_max = np.abs(d).max(axis=1)
    bad = np.flatnonzero(~np.isfinite(row_rms) | (row_rms > RMS_TOL) | (row_max > MAX_TOL))
    return float(np.nanmax(row_rms)), float(np.nanmax(row_max)), bad


def _check(label, got, ref, row0=0):
    rms, mx, bad = _errors(got, ref)
    print(f'{label}: per-frame RMS {rms:.2e}, max {mx:.2e}' + (f'; rows over the tolerance {(bad + row0)[:16].tolist()} of {len(bad)}' if len(bad) else ''))
    return rms, mx, bad


def _assert_all(failures):
    assert not failures, '; '.join(f'{label}: RMS {rms:.2e} max {mx:.2e}, first bad rows {bad[:8].tolist()}' for label, rms, mx, bad in failures)


def _layer_name(i):
    return f'c{i}' if i < 8 else f'd{i - 8}'


def _layer_shape(i, B, Tp):
    """(transposed, B, Hin, Win, C0, C1, Cout) of k4 layer i of the base-64 stage-2 U-Net (csrc/unet.cu unet_layer_shape)"""
    shapes = eng._unet_layer_shapes(2, 1, 1, 64)
    tr, cin, cout, _ = shapes[i]
    if i < 8:
        lvl, C0 = i - 1, cin
    else:
        lvl, C0 = 15 - i, cin if i == 8 else shapes[i - 1][2]
    return tr, B, Tp >> lvl, W >> lvl, C0, cin - C0, cout


def _ksplit(engine, i, B, Tp):
    """the split-K factor the wgmma kernel runs layer i with at (B, Tp): the planner's choice depends on the layer shape only"""
    tr, B, H, Wd, C0, C1, Cout = _layer_shape(i, B, Tp)
    in0 = np.zeros((B, H, Wd, C0), np.float32)
    in1 = np.zeros((B, H, Wd, C1), np.float32) if C1 else None
    Wt = np.zeros((C0 + C1, Cout, 4, 4) if tr else (Cout, C0 + C1, 4, 4), np.float32)
    _, _, ks = engine.test_conv_layer(in0, in1, Wt, np.ones(Cout, np.float32), np.zeros(Cout, np.float32), tr, 4, 2, 1, 2 if tr else 1,
                                      use_tc=1, with_ksplit=True)
    return ks


def _plan_bytes(B, Tp):
    """device bytes of one FP16 stage-2 plan (csrc/unet.cu unet_get_plan): the FP16 activations enc[0..7] and dec[0..6], the FP32 input
    and output, each rounded up to 1 KiB"""
    enc = [B * (Tp >> l) * (W >> l) * 64 * m * 2 for l, m in enumerate((1, 2, 4, 8, 8, 8, 8, 8))]
    dec = [B * (Tp >> (6 - d)) * (W >> (6 - d)) * 64 * m * 2 for d, m in enumerate((8, 8, 8, 8, 4, 2, 1))]
    io = [B * Tp * W * 4] * 2
    return sum(-(-b // 1024) * 1024 for b in enc + dec + io)


def _big_spot_members():
    """the first and last member, the member whose rows hold element 2^31 of the 64-channel full-resolution buffers, and one seeded
    other"""
    per_member = BIG_TP * W * 64
    straddle = 2 ** 31 // per_member
    other = np.random.default_rng(BIG_SEED).choice(np.delete(np.arange(1, BIG_B - 1), straddle - 1))
    return straddle, sorted({0, straddle, BIG_B - 1, int(other)})


# ---------------------------------------------------------------- the cases' own premises (no GPU)
def test_heights_cover_every_session_height():
    assert {Tp for Tp, *_ in stage2_cases()} <= set(HEIGHTS)
    assert {Tp for Tp, _, _ in BATCHED} <= set(HEIGHTS)
    for g in HEIGHTS.values():
        assert g.buckets <= 16 and 0 < g.Tp - g.Tw, g           # a window a session accepts, with padding rows
    assert BIG_B * BIG_TP * W * 64 > 2 ** 31 and BIG_B <= 64


def test_member_inputs_are_padded_distinct_and_fp16():
    for Tp, g in HEIGHTS.items():
        xs = [_member_input(Tp, j) for j in range(3)]
        for x in xs:
            assert x.shape == (Tp, W)
            assert np.array_equal(x.astype(np.float16).astype(np.float32), x)
            assert np.array_equal(x[g.Tw:], np.broadcast_to(x[:g.Tw].min(axis=0), (Tp - g.Tw, W)))
        assert not np.array_equal(xs[0], xs[1]) and not np.array_equal(xs[1], xs[2])


def test_big_case_straddles_two_to_the_31():
    straddle, members = _big_spot_members()
    per_member = BIG_TP * W * 64
    assert straddle * per_member < 2 ** 31 < (straddle + 1) * per_member
    assert {0, straddle, BIG_B - 1} < set(members)


def test_layer_shapes_match_the_plan():
    """_layer_shape restates unet_layer_shape: check it against the production layer table of test_gpu_conv_layers (Tp 384)"""
    from .test_gpu_conv_layers import PRODUCTION_LAYERS
    for name, tr, H, Wd, C0, C1, Cout, _ in PRODUCTION_LAYERS[:14]:
        i = int(name[1]) + (8 if name[0] == 'd' else 0)
        assert _layer_shape(i, 1, 384) == (tr, 1, H, Wd, C0, C1, Cout), name


# ---------------------------------------------------------------- the device against the oracle
@pytest.mark.gpu
@pytest.mark.parametrize('Tp', list(HEIGHTS))
def test_full_forward_matches_oracle(engine, full_models, Tp):
    _load_stage2(engine, full_models)
    y = engine.test_stage2_forward(_member_input(Tp, 0)[None], mode=0)
    rms, mx, bad = _check(f'full forward Tp {Tp} (Tw {HEIGHTS[Tp].Tw})', y[0], _oracle(full_models, Tp, 0))
    assert not len(bad), (rms, mx, bad[:16].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize('Tp,B,c5_splits', BATCHED)
def test_batched_forward_matches_oracle_per_member(engine, full_models, Tp, B, c5_splits):
    """B members with different data in one forward: a member that read another's rows, or a batch offset that went wrong, fails"""
    _load_stage2(engine, full_models)
    ks = {_layer_name(i): _ksplit(engine, i, B, Tp) for i in SPLIT_LAYERS}
    print(f'Tp {Tp} B {B}: split-K ' + ', '.join(f'{k} {v}' for k, v in ks.items()))
    assert (ks['c5'] > 1) == c5_splits, ks
    y = engine.test_stage2_forward(np.stack([_member_input(Tp, j) for j in range(B)]), mode=0)
    failures = []
    for j in range(B):
        rms, mx, bad = _check(f'Tp {Tp} B {B} member {j}', y[j], _oracle(full_models, Tp, j))
        if len(bad):
            failures.append((f'member {j}', rms, mx, bad))
    _assert_all(failures)


@pytest.mark.gpu
def test_largest_group_at_the_largest_window(engine, full_models):
    """64 members at Tp 1920: the 64-channel full-resolution buffers hold 4.0e9 elements, so every index into them past member 34
    row 256 needs more than 31 bits.  Each member is compared with its own batch-of-one forward (which test_full_forward_matches_oracle
    checks at this height), and the first, last, straddling and one seeded member with the oracle."""
    import torch
    n_full = BIG_B * BIG_TP * W * 64
    need = _plan_bytes(BIG_B, BIG_TP)
    free, total = torch.cuda.mem_get_info(engine.device)
    print(f'B {BIG_B} Tp {BIG_TP}: {n_full:.3e} elements per 64-channel full-resolution buffer (2^31 = {2 ** 31:.3e}); '
          f'plan {need / 2 ** 30:.2f} GiB, device free {free / 2 ** 30:.2f} of {total / 2 ** 30:.2f} GiB')
    assert n_full > 2 ** 31
    assert need < free, f'the plan needs {need} bytes and the device has {free} free of {total}'
    _load_stage2(engine, full_models)
    straddle, spot = _big_spot_members()
    print(f'member {straddle} holds element 2^31 at row {(2 ** 31 - straddle * BIG_TP * W * 64) // (W * 64)}; oracle members {spot}')
    x = np.stack([_member_input(BIG_TP, j) for j in range(BIG_B)])
    y = engine.test_stage2_forward(x, mode=0)
    failures = []
    for j in spot:
        rms, mx, bad = _check(f'B {BIG_B} member {j} vs oracle', y[j], _oracle(full_models, BIG_TP, j))
        if len(bad):
            failures.append((f'member {j} vs oracle', rms, mx, bad))
    worst = (0.0, 0.0)
    for j in range(BIG_B):
        rms, mx, bad = _errors(y[j], engine.test_stage2_forward(x[j:j + 1], mode=0)[0])
        worst = (max(worst[0], rms), max(worst[1], mx))
        if len(bad):
            print(f'B {BIG_B} member {j} vs batch of one: RMS {rms:.2e}, max {mx:.2e}, rows over the tolerance {bad[:16].tolist()}')
            failures.append((f'member {j} vs batch of one', rms, mx, bad))
    print(f'B {BIG_B}: every member vs its batch-of-one forward, worst per-frame RMS {worst[0]:.2e}, max {worst[1]:.2e}')
    _assert_all(failures)


@pytest.mark.gpu
@pytest.mark.parametrize('Tp', list(HEIGHTS))
def test_banded_and_tail_kept_rows_match_oracle(engine, full_models, Tp):
    """the kept rows of the session's banded decoder (mode 1) and of the forward that also skips the padded tail (mode 3)"""
    _load_stage2(engine, full_models)
    g = HEIGHTS[Tp]
    kb, kl = g.keep
    x = _member_input(Tp, 0)[None]
    ref = _oracle(full_models, Tp, 0)[kb:kb + kl]
    failures = []
    for mode, what in ((1, 'banded'), (3, 'tail-skipped')):
        y = engine.test_stage2_forward(x, keep=[(kb, kl)], mode=mode, tw=g.Tw if mode == 3 else 0)
        rms, mx, bad = _check(f'{what} Tp {Tp} Tw {g.Tw} rows [{kb}, {kb + kl})', y[0, kb:kb + kl], ref, row0=kb)
        if len(bad):
            failures.append((what, rms, mx, bad + kb))
    _assert_all(failures)


@pytest.mark.gpu
@pytest.mark.parametrize('gid', ['G7', 'G9'])
def test_stage2_convert_at_session_window_length(engine, full_models, gid):
    """engine.stage2_convert at T = Tw (1000 -> Tp 1024, 1919 -> Tp 1920): k_sr_colmin's column minimum over 32 and 60 row blocks, the
    U-Net, and k_sr_epilogue over every row, against oracle.nets.stage2_convert"""
    T = BY_ID[gid].Tw
    _load_stage2(engine, full_models)
    rng = np.random.default_rng(T)
    sp = np.exp(-9 + 2.5 * rng.standard_normal((T, 513))).astype(np.float32)
    ref = onets.stage2_convert(sp, _params(str(full_models['stage2_model_path'])), backend='torch')
    got = engine.stage2_convert(sp)
    assert got.shape == ref.shape and np.all(got > 0)
    rms, mx, bad = _check(f'stage2_convert T {T} (Tp {BY_ID[gid].Tp})', np.log(got.astype(np.float64)), np.log(ref.astype(np.float64)))
    assert not len(bad), (rms, mx, bad[:16].tolist())
