"""Fused stage-1 kernel (csrc/s1_fused.cu: the whole 1-D U-Net as one cluster launch) against the 16-layer wgmma sequence it replaces
and against the oracle (oracle/nets.py), base-64 model, every padded-length bucket the BASELINE configurations reach and the longer
windows of tests/session_geometry.py up to the largest a session accepts (Tw 1919, bucket 1920)."""
import numpy as np
import pytest

from oracle import nets as onets
from realtime_yukarin_b200 import synthetic

from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu


def test_fused_stage1_matches_layered_and_oracle(engine, full_models):
    ac, sr, f0c = _load(engine, full_models)
    p1 = onets.load_npz(full_models['stage1_model_path'])
    rng = np.random.default_rng(11)
    engine.set_precision('fp16')
    cluster = engine.set_stage1_fused(True)
    assert cluster >= 1, 'fused stage-1 kernel unavailable on this device'
    try:
        import os
        quick = os.environ.get('RYK_TEST_QUICK') == '1'                     # compute-sanitizer runs: two buckets are enough
        for T in ((60, 260) if quick else (3, 60, 128, 200, 260, 383, 400, 600, 640, 1000, 1100, 1500, 1919)):     # buckets 128 .. 1920
            mc = (synthetic.MC_MEAN_IN + synthetic.MC_STD_IN * rng.standard_normal((T, 9))).astype(np.float32)
            ref = onets.stage1_convert(mc, p1, backend='torch')
            engine.set_stage1_fused(True)
            fused = engine.stage1_convert(mc)
            fused2 = engine.stage1_convert(mc)
            engine.set_stage1_fused(False)
            layered = engine.stage1_convert(mc)
            e_f, e_l, e_fl = np.abs(fused - ref).max(), np.abs(layered - ref).max(), np.abs(fused - layered).max()
            print(f'stage1 T={T}: fused vs oracle {e_f:.2e}, layered vs oracle {e_l:.2e}, fused vs layered {e_fl:.2e}; cluster {cluster}')
            assert np.array_equal(fused, fused2), 'fused kernel is not deterministic'
            assert e_f < 2e-2, (T, e_f)            # the tolerance test_stage1_matches_oracle applies to the layered FP16 path
            assert e_fl < 2e-2, (T, e_fl)
    finally:
        engine.set_stage1_fused(True)
