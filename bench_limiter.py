"""Cost of the output limiter on the headline stream (precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic
voice): steps/s of device-resident ryk_session_push_device steps in blocks of --block (the device drains between blocks, as in bench.py's
sustained figure) for sessions returning 24 kHz and 48 kHz, each without the limiter and with it at a 5 ms look-ahead and a hold of 50
and of 500 ms.  The limiter runs at a gain under which the voice plays 4x over the -1 dB ceiling, so it limits on every step.

The variants alternate within each of --repeats rounds after --warmup steps each.  After the timed rounds one torch.profiler window over
--profile_steps steps of each limited session gives the three limiter kernels' device time per step, next to the synthesis stage's
other kernels.  The card's name and power limit are recorded with the numbers.

    python bench_limiter.py [--out DIR] [--steps 1000 --block 100 --warmup 30 --repeats 3 --profile_steps 20]

Prints one JSON line (and writes it to DIR/bench_limiter.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
from pathlib import Path

import numpy as np

from benchlib import (EXTRA, FS, T, alternate, bench_parser, card, device_chunks, device_pusher, emit, headline_config,
                      kernel_durations, require_cuda, synthetic_voice, throughput)

VARIANTS = [(rate, hold) for rate in (24000, 48000) for hold in (None, 50.0, 500.0)]
LOOKAHEAD_MS = 5.0
KERNELS = ('k_lim_g0', 'k_lim_min', 'k_lim_apply')


def _name(v):
    rate, hold = v
    return f'{rate // 1000}k_' + ('off' if hold is None else f'hold{int(hold)}')


def main(argv=None):
    args = bench_parser(steps=1000, block=100, warmup=30, repeats=3, profile_steps=20).parse_args(argv)
    require_cuda('bench_limiter.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_limiter_'))           # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n = round(T * FS)
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    chunks = [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(n_chunks)]
    d_in = device_chunks(x, n, n_chunks)

    # the voice's peak level over the chunks sets the gain that drives the limiter
    probe = eng.session_create(cfg, voice=voice)
    buf = np.empty(eng.session_io_geometry(probe)['max_out'])
    peak = max(float(np.max(np.abs(eng.session_push(probe, c, buf)), initial=0.0)) for c in chunks)
    eng.session_destroy(probe)
    gain = 4.0 * 10 ** (-1.0 / 20) / peak

    def make(v):
        rate, hold = v
        sid = eng.session_create(cfg, voice=voice)
        if rate != FS:
            eng.session_set_output_rate(sid, rate)
        if hold is not None:
            eng.session_limiter(sid, LOOKAHEAD_MS, hold)
            eng.session_set_limiter(sid, -1.0, gain)
        return sid
    sessions = {v: make(v) for v in VARIANTS}
    push = device_pusher(eng, d_in, max(eng.session_io_geometry(s)['max_out'] for s in sessions.values()))

    def leg(v, steps):
        return throughput(eng, lambda: push(sessions[v]), steps, args.block)
    res = alternate(VARIANTS, leg, args.steps, args.warmup, args.repeats)
    reductions = {_name(v): eng.session_limiter_stats(sessions[v]) for v in VARIANTS if v[1] is not None}

    # kernel times: one profiler window, one limited session after the other
    limited = [v for v in VARIANTS if v[1] is not None]

    def profiled_steps():
        for v in limited:
            for _ in range(args.profile_steps):
                push(sessions[v])
            eng.synchronize()
    durations = kernel_durations(eng, tmp, profiled_steps, KERNELS)
    kernels = {}
    for i, v in enumerate(limited):
        per = {}
        for name in KERNELS:
            d = durations[name][i * args.profile_steps:(i + 1) * args.profile_steps]
            per[f'{name}_us_median'] = statistics.median(d) if d else None
        per['limiter_us_per_step_median'] = sum(per[f'{name}_us_median'] or 0.0 for name in KERNELS)
        kernels[_name(v)] = per

    for sid in sessions.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)

    line = dict(card=card(), buffer_time=T, extras=EXTRA, lookahead_ms=LOOKAHEAD_MS, gain=gain, steps=args.steps, block=args.block,
                warmup=args.warmup, repeats=args.repeats,
                variants={_name(v): dict(steps_per_s=statistics.median(res[v]), steps_per_s_all=res[v]) for v in VARIANTS},
                last_step_reduction=reductions, kernels=kernels)
    emit(args.out, 'bench_limiter', line)


if __name__ == '__main__':
    main()
