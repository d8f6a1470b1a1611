"""Split-K on the wgmma convolution (conv_tc.cu) over the split factors the kernel takes: one tile's K splits run as one
thread-block cluster and meet in distributed shared memory.  The split factor is forced through the tile count the split rule
sees, on layers shaped like the bottleneck layers that split K in the stage-2 U-Net, with ragged tiles at batch 1 and 4.  Each
case matches torch within the production-layer tolerances and is bitwise the same on a second run.

The rule gives ks = 2 * SMs // tiles, at most K chunks / 8, lowered until the device holds all `tiles` clusters of ks CTAs at
once.  A factor at the K bound is forced with one tile; a smaller one with the tile counts t for which 2 * SMs // t == ks, of
which the test takes the first the device holds as clusters (on an H100 SXM no such t exists for 11: 23 clusters of 11 do not
fit, so 11 is left out)."""
import numpy as np
import pytest
import torch

from .test_gpu_conv_layers import _ref32

pytestmark = pytest.mark.gpu

# name, transposed, H, W, C0, C1, Cout, act, split factors.  K chunks of 64 channels bound the split: 128 for the 512-channel
# convolutions, 32 / 64 for the 2 x 2-tap transposed ones (at least 8 chunks per split).  Output grids are ragged against the
# tiles (e4: 5 x 10 pixels on 8 x 16 tiles; e7: 12 of 128 pixels; d3: 6 columns on 4-wide tiles).
LAYERS = [
    ('e4', 0, 11, 20, 512, 0, 512, 1, (2, 3, 4, 5, 8, 16)),
    ('e7', 0, 6, 8, 512, 0, 512, 1, (2, 6, 16)),
    ('d0', 1, 3, 4, 512, 0, 512, 2, (2, 3, 4)),
    ('d3', 1, 5, 6, 512, 512, 512, 2, (3, 5, 8)),
    ('d5', 1, 7, 10, 256, 256, 128, 2, (2, 3, 4)),
    ('d6', 1, 9, 12, 128, 128, 64, 2, (2,)),           # 64-channel N block: the other kernel configuration
]
CASES = [(layer, ks, B) for layer in LAYERS for ks in layer[-1] for B in (1, 4)]

_refs = {}


def _layer_data(layer, B):
    name, tr, H, W, C0, C1, Cout, act, _ = layer
    key = (name, B)
    if key not in _refs:
        rng = np.random.default_rng(sum(name.encode()) * 31 + B)
        in0 = rng.standard_normal((B, H, W, C0)).astype(np.float16).astype(np.float32)
        in1 = rng.standard_normal((B, H, W, C1)).astype(np.float16).astype(np.float32) if C1 else None
        Cin = C0 + C1
        shape = (Cin, Cout, 4, 4) if tr else (Cout, Cin, 4, 4)
        Wt = (rng.standard_normal(shape) / np.sqrt(Cin * 16 / (4 if tr else 1))).astype(np.float16).astype(np.float32)
        scale = rng.uniform(0.8, 1.2, Cout).astype(np.float32)
        shift = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
        _refs[key] = (in0, in1, Wt, scale, shift, _ref32(in0, in1, Wt, scale, shift, tr, act))
    return _refs[key]


@pytest.mark.parametrize('case', CASES, ids=[f'{c[0][0]}-ks{c[1]}-b{c[2]}' for c in CASES])
def test_forced_split_factor(engine, case):
    layer, ks, B = case
    name, tr, *_ = layer
    act = layer[7]
    in0, in1, Wt, scale, shift, ref = _layer_data(layer, B)
    Cin = in0.shape[3] + (in1.shape[3] if in1 is not None else 0)
    k_bound = (16 if not tr else 4) * Cin // 64 // 8
    slots = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    candidates = [1] if ks == k_bound else range(slots // (ks + 1) + 1, slots // ks + 1)

    def run(tiles):
        return engine.test_conv_layer(in0, in1, Wt, scale, shift, tr, 4, 2, 1, act, use_tc=1, ksplit_tiles=tiles, with_ksplit=True)
    for tiles in candidates:
        got, _, used = run(tiles)
        if used == ks:
            break
    assert used == ks, (name, ks, used)
    err = np.abs(got - ref)
    print(f'{name} ks {ks} B {B}: max err {err.max():.2e} rms {np.sqrt((err ** 2).mean()):.2e}')
    assert err.max() < 1.2e-2, err.max()
    assert np.sqrt((err ** 2).mean()) < 1.5e-3
    again, _, _ = run(tiles)
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), 'split-K result differs between two runs'
