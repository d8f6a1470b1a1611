"""Cost of the clock drift stage (DESIGN.md §4l): the k_drift kernel's device time per push and the host round trip of ryk_drift_push.

For each sound-card rate (24 and 48 kHz) and chunk (0.3 and 1 s), a drift stage at 250 ppm takes --warmup pushes of one chunk of
seeded noise, then:
  * one torch.profiler window over --profile_pushes pushes gives the kernel's device time per push (median);
  * --pushes further pushes, each timed on the host from the call to its return (Engine.drift_push: the copy in, the launch, the copy
    back and the wait), give the round trip (median and 90th percentile).
The card's name, power limit and SM clock are recorded with the numbers.

    python bench_drift.py [--out DIR] [--pushes 300 --warmup 20 --profile_pushes 50]

Prints one JSON line (and writes it to DIR/bench_drift.json with --out).  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from bench_f0_control import card

RATES = (24000, 48000)
CHUNKS_S = (0.3, 1.0)
PPM = 250.0


def make_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, default=None)
    ap.add_argument('--pushes', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--profile_pushes', type=int, default=50)
    return ap


def main(argv=None):
    args = make_parser().parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_drift.py needs a CUDA device')
    from torch.profiler import ProfilerActivity, profile

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
                eng.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.profile_pushes):
                        eng.drift_push(did, x)
                    eng.synchronize()
                trace = tmp / f'trace_{rate}_{n}.json'
                prof.export_chrome_trace(str(trace))
                ev = json.loads(trace.read_text())
                ev = ev['traceEvents'] if isinstance(ev, dict) else ev
                kern = [e['dur'] for e in ev if e.get('cat') == 'kernel' and e.get('ph') == 'X' and 'k_drift' in e['name']]
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
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_drift.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
