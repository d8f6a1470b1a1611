"""Cost of moving a session (ryk_session_snapshot / ryk_session_restore) on the headline stream (precision 1, 0.3 s chunks at 24 kHz,
extras 0 / 0.5 / 0, full-width synthetic voice) with every optional stage on: noise suppression, echo cancellation (32 taps), AGC,
limiter, f0 measuring with follow mode and a formant ratio.

After --steps chunks of synthetic speech (with a far end), the session is snapshotted and restored --repeats times (after --warmup
untimed rounds), alternating the two, to the same engine and to a second engine on the same device.  Reported: the blob size by
section, and the median wall time of the snapshot and of the restore, each split into its device part (enqueueing the staged copies
to their end) and its host part (the rest: waiting for the session's streams, building the session, packing, parsing, the checksum),
as ryk_snapshot_last_times measures them, beside the 300 ms chunk period.  The card's name and power limit are recorded with them.

    python bench_session_move.py [--out DIR] [--steps 20 --warmup 2 --repeats 10]

Prints one JSON line (and writes it to DIR/bench_session_move.json with --out).  Needs a CUDA device; there is no CPU path."""
import statistics
import tempfile
import time
from collections import OrderedDict
from pathlib import Path

import numpy as np

from benchlib import FS, T, bench_parser, card, emit, headline_config, require_cuda, synthetic_voice


def _stats(xs):
    return {'median': statistics.median(xs), 'min': min(xs), 'max': max(xs)}


def main(argv=None):
    args = bench_parser(steps=20, warmup=2, repeats=10).parse_args(argv)
    require_cuda('bench_session_move.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, describe_snapshot

    tmp = Path(tempfile.mkdtemp(prefix='bench_session_move_'))     # synthetic model files: never written into the tree
    engines = []
    for _ in range(2):
        e = Engine()
        e.set_precision('fp16')
        engines.append((e, synthetic_voice(e, tmp)))
    src, voice = engines[0]
    cfg = headline_config()
    n = round(T * FS)
    x = synthetic.synthetic_speech((args.steps + 1) * T, stream=3)
    far = synthetic.synthetic_speech((args.steps + 1) * T, stream=4) * 0.5
    sid = src.session_create(cfg, voice=voice)
    src.session_denoise(sid)
    src.session_denoise_learn(sid, frames=100)
    src.session_echo_cancel(sid, taps=32)
    src.session_agc(sid)
    src.session_limiter(sid)
    src.session_f0_measure(sid)
    src.session_f0_follow(sid, True, min_voiced_frames=100)
    src.session_set_formant(sid, semitones=2.0)
    buf = np.empty(src.session_io_geometry(sid)['max_out'])
    for k in range(args.steps):
        src.session_echo_reference(sid, np.ascontiguousarray(far[k * n:(k + 1) * n], np.float32))
        src.session_push(sid, np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32), buf)
    blob = src.session_snapshot(sid)
    sections = OrderedDict()
    for tag, size in describe_snapshot(blob)['sections']:
        sections[tag] = sections.get(tag, 0) + size
    result = {'bench': 'session_move', 'card': card(), 'chunk_ms': T * 1000, 'steps_before_move': args.steps, 'blob_bytes': len(blob),
              'sections_bytes': sections}
    for name, (dst, dvoice) in (('same_engine', engines[0]), ('second_engine', engines[1])):
        t = {k: [] for k in ('snapshot_wall', 'snapshot_host', 'snapshot_device', 'restore_wall', 'restore_host', 'restore_device')}
        for r in range(args.warmup + args.repeats):
            src.synchronize()
            t0 = time.perf_counter()
            blob = src.session_snapshot(sid)
            t1 = time.perf_counter()
            sh, sd = src.snapshot_last_times()
            t2 = time.perf_counter()
            b = dst.session_restore(blob, voice=dvoice)
            t3 = time.perf_counter()
            rh, rd = dst.snapshot_last_times()
            dst.session_destroy(b)
            if r >= args.warmup:
                for k, v in (('snapshot_wall', (t1 - t0) * 1e3), ('snapshot_host', sh), ('snapshot_device', sd),
                             ('restore_wall', (t3 - t2) * 1e3), ('restore_host', rh), ('restore_device', rd)):
                    t[k].append(v)
        result[name] = {k: _stats(v) for k, v in t.items()}
        result[name]['move_over_chunk'] = (statistics.median(t['snapshot_wall']) + statistics.median(t['restore_wall'])) / (T * 1000)
    emit(args.out, 'bench_session_move', result)


if __name__ == '__main__':
    main()
