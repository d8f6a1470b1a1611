"""Stage-2 row bands: a streaming session keeps only the chunk's frames of each converted window, so its stage-2 forward computes only
the decoder rows those frames depend on (unet_derive_bands in csrc/unet.cu).

* The band table of the library is checked against an independent walk that marks, row by row, what each layer reads by the
  kernels' index formulas and then rounds to the layers' tile rows.
* A banded forward on NaN-filled buffers must give finite kept rows equal to the full forward's: a row that the banded decoder
  read without computing it would carry the NaN into the output.
"""
import numpy as np
import pytest

from realtime_yukarin_b200 import engine as eng

from .session_geometry import stage2_cases

W = 512

# (Tp, keep_begin, keep_len): the session shapes at 0.1 / 0.3 / 1.0 s chunks with 0.5 s extras, 1.0 s chunks with 1.0 s extras,
# bands that touch the first and the last row, and the session geometries of tests/session_geometry.py (Tp 128 to 1920)
CASES = ([(256, 100, 20), (384, 100, 60), (512, 100, 200), (640, 200, 200), (384, 0, 60), (384, 324, 60), (128, 0, 30), (128, 90, 38)]
         + [c[:3] for c in stage2_cases()])


def _tile_rows(Win):
    """rows per 128-pixel tile of the tensor-core kernel for a transposed layer with Win input columns (conv_tc.cu tile shape)"""
    tw = 1
    while tw * 2 <= min(Win, 128):
        tw *= 2
    return 128 // tw


def _python_bands(Tp, keep_begin, keep_len):
    """[16][2] class-local rows [y0, y1) per layer, by marking the rows each computed pixel reads"""
    bands = [None] * 16
    for i in range(8):                                     # encoder: every row
        bands[i] = (0, Tp >> i)
    need = np.zeros(Tp, bool)                              # output rows of layer 15 the caller reads
    need[keep_begin:keep_begin + keep_len] = True
    for i in range(15, 7, -1):
        if i == 15:                                        # 3x3 s1 p1 conv on the CUDA-core kernel: one row per tile
            Hin, rows, th = Tp, Tp, 1
            cls = need.copy()                              # output row y is row y
        else:                                              # transposed k4 s2 p1: output row 2 m + py is class-local row m
            d = i - 8
            Hin, th = Tp >> (7 - d), _tile_rows(W >> (7 - d))
            rows = Hin
            cls = np.zeros(rows, bool)
            for r in np.flatnonzero(need):
                cls[r // 2] = True
        idx = np.flatnonzero(cls)
        y0 = idx.min() // th * th
        y1 = min(rows, -(-(idx.max() + 1) // th) * th)
        bands[i] = (y0, y1)
        need = np.zeros(Hin, bool)                         # rows of the layer below that the rounded band reads
        for m in range(y0, y1):
            if i == 15:
                reads = [m + dy - 1 for dy in range(3)]
            else:
                reads = [m + ty - 1 + py for py in (0, 1) for ty in (0, 1)]
            for iy in reads:
                if 0 <= iy < Hin:
                    need[iy] = True
    return np.array(bands, np.int32)


@pytest.mark.parametrize('Tp,kb,kl', CASES)
def test_band_table_matches_independent_walk(Tp, kb, kl):
    got = eng.stage2_row_bands(Tp, W, kb, kl)
    want = _python_bands(Tp, kb, kl)
    assert np.array_equal(got, want), (got.tolist(), want.tolist())


def test_band_table_headline_shape():
    """0.3 s chunks with 0.5 s extras: Tp 384, the chunk's frames are rows [100, 160)"""
    b = eng.stage2_row_bands(384, W, 100, 60)
    assert b[8:].tolist() == [[0, 3], [0, 6], [0, 8], [4, 12], [10, 22], [24, 41], [49, 81], [100, 160]]


def _load_stage2(engine, paths):
    from realtime_yukarin_b200.models import SuperResolution
    from realtime_yukarin_b200.params import create_sr_from_json
    SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=engine)
    engine.set_precision('fp16')


def _check_kept(full, band, band_ks, keeps):
    """kept rows finite, within the stage-2 tolerance of the full forward (log-spectrum: per-frame RMS <= 1e-2, max <= 6e-2), and
    bitwise equal to it when every layer splits K as in the full plan"""
    for j, (kb, kl) in enumerate(keeps):
        f, b, bk = full[j, kb:kb + kl], band[j, kb:kb + kl], band_ks[j, kb:kb + kl]
        assert np.isfinite(b).all() and np.isfinite(bk).all()
        d = b.astype(np.float64) - f
        rms, mx = float(np.sqrt((d ** 2).mean(axis=1)).max()), float(np.abs(d).max())
        print(f'member {j} rows [{kb}, {kb + kl}): per-frame RMS {rms:.2e}, max {mx:.2e}')
        assert rms <= 1e-2 and mx <= 6e-2, (rms, mx)
        assert np.array_equal(bk, f)


@pytest.mark.gpu
@pytest.mark.parametrize('Tp,kb,kl', CASES)
def test_banded_forward_on_nan_buffers(engine, full_models, Tp, kb, kl):
    _load_stage2(engine, full_models)
    rng = np.random.default_rng(Tp * 1000 + kb)
    x = (-9.0 + 2.5 * rng.standard_normal((1, Tp, W))).astype(np.float32)
    full = engine.test_stage2_forward(x, mode=0)
    assert np.isfinite(full).all()
    band = engine.test_stage2_forward(x, keep=[(kb, kl)], mode=1)
    band_ks = engine.test_stage2_forward(x, keep=[(kb, kl)], mode=2)
    _check_kept(full, band, band_ks, [(kb, kl)])
    # the last layer computed exactly the kept rows
    assert np.isnan(np.delete(band[0], np.s_[kb:kb + kl], axis=0)).all()


@pytest.mark.gpu
def test_group_band_is_the_hull_of_its_members(engine, full_models):
    """two members with the same 260-frame window and different extras: 0.3 s chunks with 0.5 s extras keep rows [100, 160),
    0.5 s chunks with 0.4 s extras keep rows [80, 180); the batched forward computes their hull"""
    _load_stage2(engine, full_models)
    keeps = [(100, 60), (80, 100)]
    rng = np.random.default_rng(5)
    x = (-9.0 + 2.5 * rng.standard_normal((2, 384, W))).astype(np.float32)
    full = engine.test_stage2_forward(x, mode=0)
    band = engine.test_stage2_forward(x, keep=keeps, mode=1)
    band_ks = engine.test_stage2_forward(x, keep=keeps, mode=2)
    _check_kept(full, band, band_ks, keeps)
    for j in range(2):
        assert np.isfinite(band[j, 80:180]).all()
        assert np.isnan(band[j, :80]).all() and np.isnan(band[j, 180:]).all()
