"""The U-Net layer shapes the Python side uses to check the model files of voices >= 1 (engine._unet_layer_shapes) against the
weights of model files in the Chainer layout, at the widths the tests and benchmarks use.  No GPU needed."""
import pytest

from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import _unet_layer_shapes
from realtime_yukarin_b200.models import fold_layers


@pytest.mark.parametrize('base', [16, 32, 64])
def test_layer_shapes_match_model_files(base):
    for stage, params, in_ch, out_ch in ((1, synthetic.make_stage1_params(0, base), 9, 9), (2, synthetic.make_stage2_params(0, base), 1, 1)):
        for (W, _, _), (tr, cin, cout, k) in zip(fold_layers(params), _unet_layer_shapes(stage, in_ch, out_ch, base)):
            assert tuple(W.shape[:2]) == ((cin, cout) if tr else (cout, cin)) and W.shape[-1] == k, (stage, W.shape, tr, cin, cout, k)
