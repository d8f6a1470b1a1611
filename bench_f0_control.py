"""Cost of the per-session f0 controls on the headline stream: steps per second of one device-resident session
(ryk_session_push_device, precision 1, 0.3 s chunks, extras 0 / 0.5 / 0, full-width synthetic voice) in four variants:

  off      the session as it is without the feature
  measure  ryk_session_f0_measure: one more kernel (k_f0_measure) at the end of the head of stage 1
  follow   measure + ryk_session_f0_follow: the kernel also writes the input side of the f0 map
  set      `off` with ryk_session_set_f0_map before every step: one 56-byte copy on stream C per step

Each variant is a session of its own on one engine.  A leg queues --steps steps in blocks of --block (the device drains between
blocks, as in bench.py's sustained figure) and is timed on the host clock from an idle device to an idle device; the legs of the variants
alternate within each of --repeats rounds, after --warmup steps per session.  Reported per variant: every round's steps/s, their median,
and the kernels per step from ryk_engine_launch_count.  The card's name and power limit are recorded with the numbers.

    python bench_f0_control.py [--out DIR] [--steps 3000 --block 100 --warmup 40 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_f0_control.json with --out).  Needs a CUDA device; there is no CPU path."""
import itertools
import shutil
import statistics
import tempfile
from pathlib import Path

from benchlib import (EXTRA, FS, T, alternate, bench_parser, card, device_chunks, device_pusher, emit, headline_config, require_cuda,
                      synthetic_voice, throughput)

VARIANTS = ('off', 'measure', 'follow', 'set')


def main(argv=None):
    args = bench_parser(steps=3000, block=100, warmup=40, repeats=3).parse_args(argv)
    require_cuda('bench_f0_control.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_f0_control_'))        # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n_chunks = 64
    d_in = device_chunks(synthetic.synthetic_speech((n_chunks + 1) * T, stream=0), round(T * FS), n_chunks)
    sids = {}
    for v in VARIANTS:
        sids[v] = eng.session_create(cfg, voice=voice)
        if v in ('measure', 'follow'):
            eng.session_f0_measure(sids[v])
        if v == 'follow':
            eng.session_f0_follow(sids[v], True, min_voiced_frames=200)
    push = device_pusher(eng, d_in, eng.session_io_geometry(sids['off'])['max_out'])
    base_map = eng.session_get_f0_map(sids['set'])
    semitones = itertools.cycle((-2, -1, 0, 1, 2))

    def step(v):
        if v == 'set':                            # a different map every step, so that every step stages a copy
            eng.session_set_f0_map(sids[v], target_mean=base_map['target_mean'], semitones=next(semitones))
        push(sids[v])

    def leg(v, steps):
        return throughput(eng, lambda: step(v), steps, args.block, launches=True)
    res = alternate(VARIANTS, leg, args.steps, args.warmup, args.repeats)
    measured = {v: eng.session_f0_measured(sids[v]) for v in ('measure', 'follow')}
    for sid in sids.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    rates = {v: [r for r, _ in res[v]] for v in VARIANTS}
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, block=args.block, warmup=args.warmup, repeats=args.repeats,
                variants={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=res[v][-1][1])
                          for v in VARIANTS},
                voiced_frames_counted={v: m[0] for v, m in measured.items()})
    emit(args.out, 'bench_f0_control', line)


if __name__ == '__main__':
    main()
