"""Cost of the clock drift stage (DESIGN.md §4l): the k_drift kernel's device time per push and the host round trip of ryk_drift_push.

For each sound-card rate (24 and 48 kHz) and chunk (0.3 and 1 s), a drift stage at 250 ppm takes --warmup pushes of one chunk of
seeded noise, then:
  * one torch.profiler window over --profile_pushes pushes gives the kernel's device time per push (median);
  * --pushes further pushes, each timed on the host from the call to its return (Engine.drift_push: the copy in, the launch, the copy
    back and the wait), give the round trip (median and 90th percentile).
The card's name, power limit and SM clock are recorded with the numbers.

    python bench_drift.py [--out DIR] [--pushes 300 --warmup 20 --profile_pushes 50]

Prints one JSON line (and writes it to DIR/bench_drift.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from benchlib import bench_parser, card, emit, kernel_durations, require_cuda

RATES = (24000, 48000)
CHUNKS_S = (0.3, 1.0)
PPM = 250.0


def main(argv=None):
    args = bench_parser(pushes=300, warmup=20, profile_pushes=50).parse_args(argv)
    require_cuda('bench_drift.py')
    from realtime_yukarin_b200.engine import Engine
    eng = Engine(device=0)
    tmp = Path(tempfile.mkdtemp(prefix='bench_drift_'))
    rng = np.random.default_rng(0)
    results = {}
    try:
        for rate in RATES:
            for chunk_s in CHUNKS_S:
                n = round(rate * chunk_s)
                x = rng.standard_normal(n) * 0.1
                did = eng.drift_create(n, 500.0)
                eng.drift_set(did, PPM)
                for _ in range(args.warmup):
                    eng.drift_push(did, x)

                def profiled_pushes():
                    for _ in range(args.profile_pushes):
                        eng.drift_push(did, x)
                kern = kernel_durations(eng, tmp, profiled_pushes, ['k_drift'])['k_drift']
                host = []
                for _ in range(args.pushes):
                    t0 = time.perf_counter()
                    eng.drift_push(did, x)
                    host.append((time.perf_counter() - t0) * 1e6)
                eng.drift_destroy(did)
                host.sort()
                results[f'{rate}Hz_{chunk_s}s'] = dict(
                    samples_per_push=n, outputs_per_push=n + round(n * PPM * 1e-6), kernels_seen=len(kern),
                    kernel_us_median=statistics.median(kern) if kern else None,
                    push_round_trip_us_median=statistics.median(host), push_round_trip_us_p90=host[int(0.9 * (len(host) - 1))])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        eng.close()
    line = dict(card=card(), ppm=PPM, pushes=args.pushes, warmup=args.warmup, profile_pushes=args.profile_pushes, results=results)
    emit(args.out, 'bench_drift', line)


if __name__ == '__main__':
    main()
