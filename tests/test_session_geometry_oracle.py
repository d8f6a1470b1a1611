"""The reference side of tests/test_gpu_session_geometry.py, on the CPU: the window geometries of tests/session_geometry.py reach the
shapes the table claims, StreamOracle runs at each of them, its per-step output lengths follow from the frames handed to the
synthesizer, and stream_compare.DeviceRowsOracle -- its encode and convert stages taken by an engine's per-op calls -- is bitwise the
plain StreamOracle when that engine answers with the oracle's own stages (tests/fake_engine.py)."""
import numpy as np
import pytest

from oracle import pipeline as opipe

from . import gated_speech as gs
from . import session_geometry as sg
from .fake_engine import OracleEngine
from .stream_compare import DeviceRowsOracle, run_stream

STEPS = 3
B = 1024                   # vocoder_buffer_size: the synthesizer emits whole blocks
STATS = (float(np.log(150.0)), 0.2, float(np.log(250.0)), 0.2)


def test_the_table_reaches_its_shapes():
    g = sg.BY_ID
    assert all(0 < x.Tw < x.Tp and x.Tp % 128 == 0 and x.Tp - x.Tw <= 128 and x.buckets <= sg.MAX_BUCKETS for x in sg.GEOMETRIES)
    assert all(x.n_wave == x.n_feat * x.hop and x.e_wave == x.e_enc * x.hop for x in sg.GEOMETRIES)
    assert g['G1'].n_feat == 1 and g['G1'].n_wave + 2 * g['G1'].e_wave == 120 and (g['G1'].Tw, g['G1'].Tp) == (21, 128)
    assert min(g['G2'].e_enc, g['G2'].e_conv, g['G2'].e_dec) > 0 and g['G2'].Td > g['G2'].n_feat and (g['G2'].Tw, g['G2'].Tp) == (50, 128)
    assert (g['G3'].Tw, g['G3'].Tp) == (128, 256) and g['G3'].Tw % 128 == 0
    assert (g['G4'].Tw, g['G4'].Tp) == (127, 128)
    assert g['G5'].n_feat % 2 == 1 and g['G5'].Tw % 128 == 1 and (g['G5'].Tw, g['G5'].Tp) == (129, 256)
    assert g['G6'].Tw % 128 == 0 and (g['G6'].Tw, g['G6'].Tp) == (384, 512)
    assert (g['G7'].Tw, g['G7'].Tp) == (1000, 1024) and g['G7'].e_enc > 0 and g['G7'].e_dec > 0
    assert (g['G8'].Tw, g['G8'].Tp) == (1320, 1408)
    assert (g['G9'].Tw, g['G9'].Tp) == (1919, 1920) and g['G9'].buckets == sg.MAX_BUCKETS
    assert [x.n_feat for x in sg.GEOMETRIES] == [1, 10, 128, 127, 61, 60, 200, 400, 61]
    # the first window the session refuses
    assert (sg.TOO_LONG.Tw, sg.TOO_LONG.Tp, sg.TOO_LONG.buckets) == (1920, 2048, 17)
    # stage-1 buckets above 5 and stage-2 windows of 768 rows or more
    assert max(x.buckets for x in sg.GEOMETRIES) == 16 and sum(x.Tp >= 768 for x in sg.GEOMETRIES) == 3


@pytest.mark.parametrize('geo', sg.GEOMETRIES, ids=[g.id for g in sg.GEOMETRIES])
def test_oracle_stream_and_its_device_rows_hook(small_models, geo):
    fake = OracleEngine(small_models['stage1_model_path'], small_models['stage2_model_path'])
    fake.f0_set_stats(*STATS)
    cfg = opipe.PathConfig()
    x = gs.stream_with_pauses(seconds=(STEPS + 1) * geo.buffer_time + 0.1)
    chunks = [x[k * geo.n_wave:(k + 1) * geo.n_wave] for k in range(STEPS)]
    orc = opipe.StreamOracle(cfg, fake.p1, fake.p2, STATS, buffer_time=geo.buffer_time, extra=geo.extra, backend='torch')
    outs, rows, total = [], [], 0
    for k, c in enumerate(chunks):
        y = orc.push(c)
        outs.append(y)
        rows.append({kk: orc.last['converted'][kk] for kk in ('f0', 'sp', 'ap')})
        assert all(len(v) == geo.n_feat for v in rows[-1].values()), k
        # whole blocks, as many as end before the last pulse placed so far, which lies within fft_size samples of the end of the
        # (k + 1) Td frames handed to the synthesizer
        pulses = orc.synth.pulses()[0]
        end = (k + 1) * geo.Td * geo.hop
        total += len(y)
        assert len(y) % B == 0, k
        if len(pulses):
            assert end - 1024 < pulses[-1] <= end and total == B * ((int(pulses[-1]) - 1) // B), (k, total, int(pulses[-1]), end)
        else:
            assert total == 0, k
    plain_pulses, _, plain_vuv = orc.synth.pulses()
    hooked = run_stream(DeviceRowsOracle(fake, cfg, geo.buffer_time, geo.extra), chunks)
    print(f'{geo.id}: n_feat {geo.n_feat} Tw {geo.Tw} Tp {geo.Tp} buckets {geo.buckets} Td {geo.Td}; samples per step '
          f'{[len(y) for y in outs]}, pulses {len(plain_pulses)}')
    assert [len(y) for y in hooked.outs] == [len(y) for y in outs]
    assert all(np.array_equal(a, b) for a, b in zip(hooked.outs, outs))
    for a, b in zip(hooked.rows, rows):
        for kk in ('f0', 'sp', 'ap'):
            assert a[kk].shape == b[kk].shape and np.array_equal(a[kk], b[kk]), kk
    assert np.array_equal(hooked.pulses, plain_pulses) and np.array_equal(hooked.vuv, plain_vuv)
