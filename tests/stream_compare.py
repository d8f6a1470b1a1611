"""A streaming session against the FP64 / torch-CPU oracle stream -- TEST INFRASTRUCTURE.

  * DeviceRowsOracle: the oracle's window bookkeeping (oracle.pipeline.StreamOracle) and synthesizer over the device's per-op rows --
    ryk_world_analyze on each encode window (the session's analysis kernels) and ryk_convert_window on each convert window -- at any
    geometry.  Its converted rows are the f0 / sp / ap rows a session hands its synthesizer, rebuilt through the per-op calls.
  * compare_stream: per-step lengths and whole-stream / per-chunk sample RMSE.
  * compare_stream_pulse_aware: the tight comparison, made in the parts that can each be held tight (see its docstring).
"""
from dataclasses import dataclass
from typing import List

import numpy as np

from oracle import pipeline as opipe
from oracle import world as oworld

from .test_gpu_headline_parity import _rmse, _waveform_spectral_distance

CFG = opipe.PathConfig()
SP_TOL = {('small', 'fp32'): (2e-3, None), ('small', 'fp16'): (3e-2, 0.25), ('full', 'fp16'): (1e-2, 6e-2)}     # (per-frame log-L2, max)
PULSES_PER_MOVE = 4000       # one moved pulse allowed per this many pulses (or part of it): one in 3416 seen at 0.3 s chunks


def logspec(a, b, rows):
    """(largest per-frame RMS, max) of ln a - ln b over `rows`"""
    if not rows.any():
        return 0.0, 0.0
    d = np.log(np.asarray(a, np.float64)[rows]) - np.log(np.asarray(b, np.float64)[rows])
    return float(np.sqrt((d ** 2).mean(axis=1)).max()), float(np.abs(d).max())


class DeviceRowsOracle(opipe.StreamOracle):
    """StreamOracle with its encode and convert stages taken by the engine's per-op calls at the engine's current precision."""

    def __init__(self, engine, cfg, buffer_time, extra):
        super().__init__(cfg, None, None, None, buffer_time=buffer_time, extra=extra)
        self.engine = engine

    def _extract(self, win):
        c = self.cfg
        a = self.engine.world_analyze(win, c.fs, c.frame_period, c.f0_floor, c.f0_ceil, c.fft_length, c.order, c.alpha)
        return dict(f0=a['f0'][:, None], sp=a['sp'], ap=a['ap'], mc=a['mc'], voiced=a['voiced'][:, None])

    def _convert(self, wave, feat):
        c = self.cfg
        out = self.engine.convert_window(wave, c.fs, c.fft_length, c.hop, c.threshold_db, feat['f0'], feat['ap'], feat['mc'],
                                         feat['voiced'], c.order, c.alpha, c.fft_length)
        return dict(out, f0=out['f0'][:, None], voiced=out['voiced'][:, None])


@dataclass
class StreamRun:
    outs: List[np.ndarray]      # samples per step, NaN scrubbed
    rows: List[dict]            # the f0 (n, 1) / sp / ap rows the synthesizer was given per step
    pulses: np.ndarray          # sample index of every pulse the synthesizer placed
    vuv: np.ndarray             # and its voicing


def run_stream(orc, chunks):
    outs, rows = [], []
    for c in chunks:
        outs.append(orc.push(c))
        rows.append({k: orc.last['converted'][k] for k in ('f0', 'sp', 'ap')})
    idx, _, vuv = orc.synth.pulses()
    return StreamRun(outs, rows, idx, vuv)


def compare_stream(label, outs, refs, rmse_tol, chunk_tol, lsd_tol=None, silent_ok=False):
    assert [len(o) for o in outs] == [len(r) for r in refs], label
    per = [_rmse(o, r) if len(r) else 0.0 for o, r in zip(outs, refs)]
    y, r = np.concatenate(outs), np.concatenate(refs)
    assert len(r) > 0 and np.isfinite(y).all()
    rmse, rms, lsd = _rmse(y, r), float(np.sqrt(np.mean(r ** 2))), _waveform_spectral_distance(y, r)
    print(f'{label}: {len(y)} samples, sample RMSE {rmse:.3e} (signal RMS {rms:.3e}), worst chunk {max(per):.3e} (step {int(np.argmax(per))}), '
          f'log-STFT distance {lsd:.3e}')
    if max(per) > chunk_tol:
        print('  per-chunk (step, rmse):', [(k, f'{e:.1e}') for k, e in enumerate(per) if e > chunk_tol / 10])
    assert silent_ok or rms > 1e-2
    assert rmse <= rmse_tol, (label, rmse)
    assert max(per) <= chunk_tol, (label, max(per))
    assert lsd_tol is None or lsd <= lsd_tol, (label, lsd)


def compare_stream_pulse_aware(label, outs, ref, dev, models, precision, lsd_tol=None):
    """A session's per-step samples `outs` against the oracle stream `ref` where one sample of pulse placement may differ; `dev` is
    the DeviceRowsOracle run on the same chunks at the session's precision.

    The synthesizer places a pulse at the first sample after its phase crosses a multiple of 2 pi: a discrete function of the last bits of the
    f0 history (DESIGN.md section 5, lesson 2).  The device's converted f0 is the oracle's to FP32 rounding, one ulp apart on about one
    voiced frame in a hundred, which is enough to move a pulse that lands on a sample boundary by one sample; the two outputs then differ
    by up to the pulse's amplitude over that pulse's response (fft_size samples) and nowhere else.  So the comparison is made in the parts
    that can each be held tight:
      * the rows the synthesizer is given (rebuilt through the per-op calls) equal the oracle's to the window tolerances, voicing exactly,
        f0 to 1e-6 relative, ap to 1e-6;
      * the oracle's own synthesizer, fed those rows, places the same pulses as on the oracle's rows with the same voicing, except that
        at most one in PULSES_PER_MOVE of them (and at least one) sits one sample later or earlier (printed);
      * FP32: the session's samples are that synthesizer's samples to 1e-9 everywhere, the moved pulses included -- the session's graphs,
        bucket switch and hand-off slots add nothing of their own;
      * outside the response of a moved pulse the session equals the oracle stream: 1e-6 per sample in FP32, the headline tolerances in FP16.
    -> the number of moved pulses"""
    fft = oworld.cheaptrick_fft_size(CFG.fs)
    assert [len(d['f0']) for d in dev.rows] == [len(o['f0']) for o in ref.rows], label
    worst = dict(sp=0.0, sp_max=0.0, ap=0.0)
    ulps = 0
    for k, (d, o) in enumerate(zip(dev.rows, ref.rows)):
        df0, of0 = d['f0'].ravel(), o['f0'].ravel()
        assert np.array_equal(df0 != 0, of0 != 0), (label, k)
        assert np.allclose(df0, of0, rtol=1e-6, atol=0), (label, k)
        ulps += int((df0.view(np.uint32) != of0.view(np.uint32)).sum())
        l2, mx = logspec(d['sp'], o['sp'], np.ones(len(of0), bool))
        worst['sp'], worst['sp_max'] = max(worst['sp'], l2), max(worst['sp_max'], mx)
        if len(of0):
            worst['ap'] = max(worst['ap'], float(np.abs(d['ap'] - o['ap']).max()))
    l2_tol, mx_tol = SP_TOL[(models, precision)]
    assert worst['sp'] < l2_tol and (mx_tol is None or worst['sp_max'] < mx_tol) and worst['ap'] <= 1e-6, (label, worst)
    idx_o, vuv_o, idx_d, vuv_d = ref.pulses, ref.vuv, dev.pulses, dev.vuv
    assert len(idx_o) == len(idx_d) and np.array_equal(vuv_o, vuv_d), label
    moved = np.flatnonzero(idx_o != idx_d)
    allowed = max(1, -(-len(idx_o) // PULSES_PER_MOVE))
    print(f'{label}: synthesizer rows vs oracle: f0 differs by one ulp on {ulps} frames, sp per-frame log-L2 {worst["sp"]:.2e} '
          f'(max {worst["sp_max"]:.2e}), ap {worst["ap"]:.1e}; {len(idx_o)} pulses, moved (at most {allowed}): '
          f'{[(int(j), int(idx_o[j]), int(idx_d[j])) for j in moved]} (pulse, oracle sample, sample on the device rows)')
    assert len(moved) <= allowed and (np.abs(idx_o[moved] - idx_d[moved]) == 1).all(), (label, moved)
    refs = ref.outs
    assert [len(o) for o in outs] == [len(r) for r in refs] == [len(o) for o in dev.outs], label
    y, r, yd = np.concatenate(outs), np.concatenate(refs), np.concatenate(dev.outs)
    assert np.isfinite(y).all() and float(np.sqrt(np.mean(r ** 2))) > 1e-2
    if precision == 'fp32':
        print(f'{label}: session vs the oracle synthesizer on the device rows: max {np.abs(y - yd).max():.2e}')
        assert np.abs(y - yd).max() <= 1e-9, label
    inside = np.zeros(len(r), bool)
    for j in moved:
        inside[max(0, int(min(idx_o[j], idx_d[j])) - fft):int(max(idx_o[j], idx_d[j])) + fft] = True
    if len(moved):
        print(f'{label}: inside the moved pulses\' responses: {int(inside.sum())} samples, max difference {np.abs(y - r)[inside].max():.2e}; '
              f'over the whole stream: sample RMSE {_rmse(y, r):.3e}, worst chunk {max(_rmse(o, q) for o, q in zip(outs, refs) if len(q)):.3e}')
        assert float(np.abs(r[inside]).max()) > 0 and np.abs(y - r)[inside].max() <= 2 * float(np.abs(r).max()), label
    assert _rmse(y, r) <= 1e-3, (label, _rmse(y, r))                             # the moved pulses included
    y_out = np.where(inside, r, y)                                               # everything else
    if precision == 'fp32':
        print(f'{label}: outside them: max {np.abs(y_out - r).max():.2e}')
        assert np.abs(y_out - r).max() <= 1e-6, label
    bounds = np.cumsum([0] + [len(o) for o in outs])
    compare_stream(label + ' (outside a moved pulse)', [y_out[a:b] for a, b in zip(bounds[:-1], bounds[1:])], refs, 1e-3,
                   1e-3 if precision == 'fp32' else 2e-3, lsd_tol=lsd_tol)
    return len(moved)
