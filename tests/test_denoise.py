"""The FP64 reference of the input noise suppression (DESIGN.md DECIDE N1-N3), without a GPU:

  * at reduction 0 (or without a profile) it reconstructs its input to rounding: sqrt-Hann squared at hop N / 4 sums to 2;
  * fed in chunks with its state carried it is exactly the whole-signal filter, whatever the chunk length;
  * learning averages P over the frames it was asked for, and the profile applies from the next step;
  * on the golden speech after 1 s of seeded white or pink noise it raises the SNR and removes the noise in the pause.
"""
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import wave_io

from . import denoise_oracle as O

GOLDEN = Path(__file__).parent / 'golden' / 'audioA_24k_4s.wav'
LEAD = 24000                     # 1 s of noise before the speech


def _speech():
    x, fs = wave_io.read_wav(GOLDEN)
    assert fs == 24000
    return np.asarray(x, np.float64)


def _noise(kind, n, seed=0):
    nz = np.random.default_rng(seed).standard_normal(n)
    if kind == 'pink':
        F = np.fft.rfft(nz)
        f = np.arange(len(F), dtype=np.float64)
        f[0] = 1.0
        nz = np.fft.irfft(F / np.sqrt(f), n)
    return nz


def _noisy(kind, snr_db, seed=0):
    """(clean, noisy float32): LEAD samples of noise alone, then the golden speech plus the noise at snr_db over the speech"""
    x = _speech()
    nz = _noise(kind, len(x) + LEAD, seed)
    scale = np.sqrt(np.mean(x ** 2) / np.mean(nz ** 2) / 10 ** (snr_db / 10))
    clean = np.concatenate([np.zeros(LEAD), x])
    return clean, (clean + scale * nz).astype(np.float32)


def test_reduction_zero_reconstructs_the_input():
    x = np.random.default_rng(3).standard_normal(20000).astype(np.float32)
    phi = O.frame_powers(x, 3, 50).mean(axis=0)
    for reduction, profile in ((0.0, phi), (20.0, None), (40.0, np.zeros(O.NB))):
        o = O.DenoiseOracle(reduction, profile)
        o.push(np.concatenate([x, np.zeros(O.D, np.float32)]))
        rebuilt = 0.5 * o.acc[O.D:O.D + len(x)]
        err = float(np.max(np.abs(rebuilt - x.astype(np.float64))))
        assert err < 1e-14, (reduction, err)
        assert np.array_equal(O.denoise(x, reduction, profile), x), reduction


@pytest.mark.parametrize('chunk', [7200, 2400, 1337, 127])
def test_chunks_with_carried_state_are_the_whole_signal(chunk):
    _, noisy = _noisy('white', 10.0, seed=1)
    x = noisy[:60000]
    phi = O.frame_powers(x, 3, 100).mean(axis=0)
    whole = O.denoise(x, 20.0, phi)
    o = O.DenoiseOracle(20.0, phi)
    pad = np.concatenate([x, np.zeros(O.D + chunk, np.float32)])
    outs = [o.push(pad[i:i + chunk]) for i in range(0, len(x) + O.D, chunk)]
    y = np.concatenate(outs)
    assert np.array_equal(y[:O.D], np.zeros(O.D, np.float32))
    assert np.array_equal(y[O.D:O.D + len(x)], whole)
    assert not np.array_equal(whole, x)


def test_learning_is_the_mean_over_the_frames_and_applies_from_the_next_step():
    _, noisy = _noisy('pink', 10.0, seed=2)
    n, frames = 7200, 188
    chunks = [noisy[i:i + n] for i in range(0, 12 * n, n)]
    o = O.DenoiseOracle(20.0)
    outs = [o.push(chunks[0])]
    first = o.frames_done
    o.learn(frames)
    assert o.frames_left() == frames
    left = []
    while not left or left[-1]:
        outs.append(o.push(chunks[len(outs)]))
        left.append(o.frames_left())
    assert left == sorted(left, reverse=True) and len(left) == 4       # 188 frames at 56.25 per step: the fourth step finishes
    k = len(outs)
    learned = o.profile()
    np.testing.assert_array_equal(learned, O.frame_powers(noisy, first, frames).mean(axis=0))
    outs.append(o.push(chunks[k]))
    # the same stream with the learned profile set by hand in front of step k: equal everywhere, and step k differs from no profile
    ref, plain = O.DenoiseOracle(20.0), O.DenoiseOracle(20.0)
    refs = [ref.push(c) for c in chunks[:k]]
    ref.set_profile(learned)
    refs.append(ref.push(chunks[k]))
    assert all(np.array_equal(a, b) for a, b in zip(outs, refs))
    plains = [plain.push(c) for c in chunks[:k + 1]]
    assert all(np.array_equal(a, b) for a, b in zip(outs[:k], plains[:k]))
    assert not np.array_equal(outs[k], plains[k])
    # a profile set cancels a learning in progress
    o.learn(500)
    o.push(chunks[k + 1])
    o.set_profile(np.ones(O.NB))
    assert o.frames_left() == 0
    o.push(chunks[k + 2])
    assert o.learn_left == 0 and np.array_equal(o.phi, np.ones(O.NB))


@pytest.mark.parametrize('kind', ['white', 'pink'])
def test_quality_on_speech_in_noise(kind):
    seg = slice(LEAD, None)
    report = []
    for snr_db, min_gain in ((10.0, 5.0), (0.0, 7.0)):
        clean, noisy = _noisy(kind, snr_db)
        phi = O.frame_powers(noisy, 3, 150).mean(axis=0)       # 150 frames of noise alone
        z = O.denoise(noisy, 20.0, phi).astype(np.float64)
        snr_in = 10 * np.log10(np.sum(clean[seg] ** 2) / np.sum((noisy[seg] - clean[seg]) ** 2))
        snr_out = 10 * np.log10(np.sum(clean[seg] ** 2) / np.sum((z[seg] - clean[seg]) ** 2))
        residual = 10 * np.log10(np.mean(z[2000:LEAD] ** 2) / np.mean(noisy[2000:LEAD].astype(np.float64) ** 2))
        report.append(f'{kind} noise at {snr_in:.1f} dB: SNR {snr_out:.1f} dB after the filter, noise alone {residual:.1f} dB')
        assert snr_out - snr_in >= min_gain
        assert residual <= -15.0
    print('; '.join(report))
