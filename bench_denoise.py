"""Cost of the input noise suppression on the headline stream: steps per second of one device-resident session
(ryk_session_push_device, precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic voice) in three variants:

  off      the session without the filter
  profile  ryk_session_denoise with a noise profile set before the first step (reduction 20 dB)
  learn    ryk_session_denoise learning a profile on every step (one learning longer than the run)

Each variant is a session of its own on one engine, created with RYK_STAGE_TIMES=1.  A leg queues --steps steps in blocks of --block
(the device drains between blocks, as in bench.py's sustained figure) and is timed on the host clock from an idle device to an idle
device; the legs of the variants alternate within each of --repeats rounds, after --warmup steps per session.  Reported per variant:
every round's steps/s and their median, the kernels per step from ryk_engine_launch_count, and the median device time of the gate stage
(input resampler, filter, wave slides) over the last 8 steps of every leg.  The card's name and power limit are recorded with the numbers.

    python bench_denoise.py [--out DIR] [--steps 3000 --block 100 --warmup 40 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_denoise.json with --out).  Needs a CUDA device; there is no CPU path."""
import os
import shutil
import statistics
import tempfile
from pathlib import Path

import numpy as np

from benchlib import (EXTRA, FS, T, alternate, bench_parser, card, device_chunks, device_pusher, emit, headline_config, require_cuda,
                      synthetic_voice, throughput)

VARIANTS = ('off', 'profile', 'learn')


def main(argv=None):
    args = bench_parser(steps=3000, block=100, warmup=40, repeats=3).parse_args(argv)
    require_cuda('bench_denoise.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_denoise_'))           # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    x = (x + 0.01 * np.random.default_rng(0).standard_normal(len(x))).astype(np.float32)
    d_in = device_chunks(x, round(T * FS), n_chunks)
    prev = os.environ.get('RYK_STAGE_TIMES')
    os.environ['RYK_STAGE_TIMES'] = '1'
    try:
        sids = {v: eng.session_create(cfg, voice=voice) for v in VARIANTS}
    finally:
        if prev is None:
            os.environ.pop('RYK_STAGE_TIMES', None)
        else:
            os.environ['RYK_STAGE_TIMES'] = prev
    for v in ('profile', 'learn'):
        eng.session_denoise(sids[v])
    eng.session_set_noise_profile(sids['profile'], np.full(257, 0.01 ** 2 * 256.0))    # white noise at 0.01 RMS: sum(w^2) = 256
    eng.session_denoise_learn(sids['learn'], frames=10 ** 12)
    push = device_pusher(eng, d_in, eng.session_io_geometry(sids['off'])['max_out'])

    def leg(v, steps):
        rate, kernels = throughput(eng, lambda: push(sids[v]), steps, args.block, launches=True)
        start, end = eng.session_stage_times(sids[v])
        return rate, kernels, float(np.median(end[:, 0] - start[:, 0]))
    res = alternate(VARIANTS, leg, args.steps, args.warmup, args.repeats)
    left = eng.session_noise_profile(sids['learn'])[1]
    for sid in sids.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    rates = {v: [r for r, _, _ in res[v]] for v in VARIANTS}
    gate = {v: [g for _, _, g in res[v]] for v in VARIANTS}
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, block=args.block, warmup=args.warmup, repeats=args.repeats,
                learn_frames_left=left,
                variants={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=res[v][-1][1],
                                  gate_ms=statistics.median(gate[v]), gate_ms_all=gate[v])
                          for v in VARIANTS})
    emit(args.out, 'bench_denoise', line)


if __name__ == '__main__':
    main()
