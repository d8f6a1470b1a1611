"""Cost of the pitch correction on the headline stream (precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic
voice): steps/s of device-resident ryk_session_push_device steps in blocks of --block (the device drains between blocks, as in bench.py's
sustained figure) for a session without the correction and with it (D major, 30 ms retune, amount 1); then the same two for a group of
8 members (ryk_group_push_device).

The variants alternate within each of --repeats rounds after --warmup steps each.  After the timed rounds one torch.profiler window
over --profile_steps steps of the session with the correction gives k_pitch's device time per step: its recursion runs on one thread
over the 60 frames of a 0.3 s step, on stream D ahead of the synthesizer.  The card's name and power limit are recorded with the
numbers.

    python bench_pitch.py [--out DIR] [--steps 1000 --block 100 --warmup 30 --repeats 3 --profile_steps 20]

Prints one JSON line (and writes it to DIR/bench_pitch.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
from pathlib import Path

from benchlib import (EXTRA, FS, T, alternate, bench_parser, card, device_chunks, device_pusher, emit, headline_config,
                      kernel_durations, require_cuda, synthetic_voice, throughput)

VARIANTS = ('off', 'pitch')
MEMBERS = 8
KERNEL = 'k_pitch'
SETTINGS = dict(key='D', scale='major', a4_hz=440.0, retune_ms=30.0, amount=1.0)


def main(argv=None):
    args = bench_parser(steps=1000, block=100, warmup=30, repeats=3, profile_steps=20).parse_args(argv)
    require_cuda('bench_pitch.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_pitch_'))               # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n_chunks = 64
    d_in = device_chunks(synthetic.synthetic_speech((n_chunks + 1) * T, stream=0), round(T * FS), n_chunks)

    def make(v):
        sid = eng.session_create(cfg, voice=voice)
        if v == 'pitch':
            eng.session_pitch_correct(sid)
            eng.session_set_pitch_correct(sid, **SETTINGS)
        return sid
    sessions = {v: make(v) for v in VARIANTS}
    groups = {v: eng.group_create([make(v) for _ in range(MEMBERS)]) for v in VARIANTS}
    push = device_pusher(eng, d_in, eng.session_io_geometry(sessions['off'])['max_out'], MEMBERS)
    legs = [(kind, v) for kind in ('single', 'group') for v in VARIANTS]

    def leg(kind_v, steps):
        kind, v = kind_v
        target = sessions[v] if kind == 'single' else groups[v]
        return throughput(eng, lambda: push(target, group=kind == 'group'), steps, args.block)
    res = alternate(legs, leg, args.steps, args.warmup, args.repeats)
    meters = {v: eng.session_pitch_stats(sessions[v]) for v in VARIANTS if v != 'off'}

    # kernel time: one profiler window over the session with the correction
    profiled = [v for v in VARIANTS if v != 'off']

    def profiled_steps():
        for v in profiled:
            for _ in range(args.profile_steps):
                push(sessions[v])
            eng.synchronize()
    pitch_us = kernel_durations(eng, tmp, profiled_steps, [KERNEL])[KERNEL]
    kernels = {}
    for i, v in enumerate(profiled):
        d = pitch_us[i * args.profile_steps:(i + 1) * args.profile_steps]
        kernels[v] = {f'{KERNEL}_us_median': statistics.median(d) if d else None, f'{KERNEL}_us_max': max(d) if d else None}

    for gid in groups.values():
        members = eng.group_members(gid)
        eng.group_destroy(gid)
        for sid in members:
            eng.session_destroy(sid)
    for sid in sessions.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)

    line = dict(card=card(), buffer_time=T, extras=EXTRA, members=MEMBERS, settings=SETTINGS, steps=args.steps, block=args.block,
                warmup=args.warmup, repeats=args.repeats,
                legs={f'{kind}_{v}': dict(steps_per_s=statistics.median(r), steps_per_s_all=r) for (kind, v), r in res.items()},
                last_step_meter={v: dict(voiced=m[0], mean_cents=m[1], max_cents=m[2]) for v, m in meters.items()}, kernels=kernels)
    emit(args.out, 'bench_pitch', line)


if __name__ == '__main__':
    main()
