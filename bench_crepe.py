"""Cost of the CREPE f0 mode of the streaming session on one GPU.

One 1-stream session at 0.3 s chunks (extras 0 / 0.5 / 0, full-width synthetic U-Nets) per leg: DIO (reference point), CREPE tiny and
CREPE full, each in precision 0 (FP32 everywhere) and 1 (FP16 tensor-core U-Nets).  Each leg creates its session, warms up its graphs,
then times --steps device-resident steps with CUDA events on the engine's stopwatch; the legs alternate over --rounds rounds so that
clock and neighbour drift spreads over all of them.  Reported per leg: ms per step and chunks/s (median over rounds) and the device
time of the analysis stage (stage 1 of ryk_session_stage_times, mean over the last 8 steps), next to the CREPE network's arithmetic per
analysis window computed from the layer shapes.  Also the CREPE network's own device time per window with each conv back-end
(and the FLOP/s that makes), and the device memory one session takes with each f0 front-end.  The card's name and power limit are recorded with the numbers.

    python bench_crepe.py --out DIR [--steps 200 --warmup 20 --rounds 3]

Writes DIR/bench_crepe.json and prints it.  Needs a CUDA device; there is no CPU path."""
import os
import shutil
import statistics
import tempfile
from pathlib import Path

import numpy as np

from benchlib import (EXTRA, FS, T, bench_parser, card, device_chunks, device_pusher, emit, headline_config, require_cuda, stopwatch_ms,
                      synthetic_builtin)

FILTERS, WIDTHS = [32, 4, 4, 4, 8, 16], [512, 64, 64, 64, 64, 64]
LEGS = [('dio', None, 'fp32'), ('dio', None, 'fp16'), ('crepe', 'tiny', 'fp32'), ('crepe', 'tiny', 'fp16'),
        ('crepe', 'full', 'fp32'), ('crepe', 'full', 'fp16')]


def crepe_flop_per_frame(capacity):
    """Multiply-adds x 2 of conv layers 1..6 and the dense layer for one 1024-sample frame."""
    m = {'tiny': 4, 'small': 8, 'medium': 16, 'large': 24, 'full': 32}[capacity]
    cout = [f * m for f in FILTERS]
    flop, w = 2 * 256 * 512 * cout[0], 128        # layer 1: 256 outputs of a k512 window; then MaxPool halves the width
    for l in range(1, 6):
        flop += 2 * w * WIDTHS[l] * cout[l - 1] * cout[l]
        w //= 2
    return flop + 2 * 4 * cout[5] * 360


def main():
    args = bench_parser(required_out=True, steps=200, warmup=20, rounds=3).parse_args()
    require_cuda('bench_crepe.py')
    import torch
    os.environ['RYK_STAGE_TIMES'] = '1'
    from realtime_yukarin_b200 import crepe, synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_crepe_'))       # synthetic model files: never written into the tree
    eng = Engine()
    synthetic_builtin(eng, tmp)
    weights = {}
    for c in ('tiny', 'full'):
        (tmp / c).mkdir()
        weights[c] = synthetic.write_crepe_model(tmp / c, seed=1, capacity=c)
    n = round(T * FS)
    total = args.warmup + args.steps
    x = synthetic.synthetic_speech((total + 1) * T, stream=0)
    d_in = device_chunks(x, n, total)
    out_cap = (n // 1024 + 5) * 1024 + 8192
    cfg = headline_config()

    def leg(method, capacity, precision):
        if capacity is not None:
            crepe.load_crepe_model(weights[capacity], eng)
        eng.set_precision(precision)
        eng.set_f0_method(method)
        sid = eng.session_create(cfg)
        eng.set_f0_method('dio')
        push = device_pusher(eng, d_in, out_cap)
        ms = stopwatch_ms(eng, lambda: push(sid), args.warmup, args.steps)
        st, en = eng.session_stage_times(sid)
        eng.session_destroy(sid)
        return ms / args.steps, float((en[:, 1] - st[:, 1]).mean())

    results = {leg_: [] for leg_ in LEGS}
    leg(*LEGS[-1])                                   # first-use costs (module load, cuFFT plans) outside the rounds
    for _ in range(args.rounds):
        for leg_ in LEGS:
            results[leg_].append(leg(*leg_))
    F = round((T + 2 * EXTRA[0]) * 200) + 1          # CREPE frames per 0.3 s encode window (= WORLD frames)
    # the CREPE network alone on one window (61 frames), per conv back-end: device time per run from CUDA events over 20 runs
    x16 = np.ascontiguousarray(x[:(F - 1) * 80], dtype=np.float32)
    network = []
    for capacity in ('tiny', 'full'):
        crepe.load_crepe_model(weights[capacity], eng)
        flop = crepe_flop_per_frame(capacity) * F
        for backend in (0, 1):
            crepe.run_test_network(eng, backend, x16, 5.0, repeat=3)
            ms = crepe.run_test_network(eng, backend, x16, 5.0, repeat=20)[3]
            network.append(dict(capacity=capacity, conv_backend=['fp32 cuda cores', '3xtf32 tensor cores'][backend], ms_per_window=ms,
                                tflops=flop / ms / 1e9))
    # device memory one session takes, by f0 front-end (precision 1): free memory before creation minus after
    footprint = {}
    for name, capacity in (('dio', None), ('crepe-tiny', 'tiny'), ('crepe-full', 'full')):
        if capacity is not None:
            crepe.load_crepe_model(weights[capacity], eng)
        eng.set_precision('fp16')
        eng.set_f0_method('dio' if capacity is None else 'crepe')
        eng.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        sid = eng.session_create(cfg)
        eng.synchronize()
        footprint[name] = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
        eng.set_f0_method('dio')
        eng.session_destroy(sid)
    rows = []
    for (method, capacity, precision), v in results.items():
        ms = statistics.median(a for a, _ in v)
        rows.append(dict(f0=method if capacity is None else f'crepe-{capacity}', precision=precision, ms_per_step=ms, chunks_per_s=1000.0 / ms,
                         ms_per_step_all=[a for a, _ in v], analysis_stage_ms=statistics.median(b for _, b in v),
                         crepe_gflop_per_window=None if capacity is None else crepe_flop_per_frame(capacity) * F / 1e9))
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, warmup=args.warmup, rounds=args.rounds, frames_per_window=F,
                note='CREPE convolutions: FP32 CUDA cores (conv_direct.cu) in precision 0, 3xTF32 tensor cores (crepe_tc.cu) in precision 1',
                legs=rows, crepe_network=network, session_mib=footprint)
    shutil.rmtree(tmp, ignore_errors=True)
    emit(args.out, 'bench_crepe', line)


if __name__ == '__main__':
    main()
