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
import argparse
import json
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from bench_f0_control import EXTRA, FS, T, card

VARIANTS = ('off', 'pitch')
MEMBERS = 8
KERNEL = 'k_pitch'
SETTINGS = dict(key='D', scale='major', a4_hz=440.0, retune_ms=30.0, amount=1.0)


def make_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, default=None)
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--block', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--profile_steps', type=int, default=20)
    return ap


def main(argv=None):
    args = make_parser().parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_pitch.py needs a CUDA device')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import load_voice

    tmp = Path(tempfile.mkdtemp(prefix='bench_pitch_'))               # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    paths = synthetic.write_synthetic_models(tmp / 'v0', seed=0)
    voice = eng.voice_create()
    load_voice(eng, voice, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path', 'target_statistics_path')})
    cfg = SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                        encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                        vocoder_buffer_size=1024)
    n = round(T * FS)
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0).astype(np.float32)
    chunks = [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(n_chunks)]
    d_in = torch.from_numpy(np.stack(chunks)).cuda()

    def make(v):
        sid = eng.session_create(cfg, voice=voice)
        if v == 'pitch':
            eng.session_pitch_correct(sid)
            eng.session_set_pitch_correct(sid, **SETTINGS)
        return sid
    sessions = {v: make(v) for v in VARIANTS}
    groups = {v: eng.group_create([make(v) for _ in range(MEMBERS)]) for v in VARIANTS}
    cap = eng.session_io_geometry(sessions['off'])['max_out']
    ring = 8                                      # distinct output slots: consecutive steps are in flight together
    d_out = torch.empty((ring, MEMBERS, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((ring, MEMBERS, 1), dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    step_no = {}

    def push_device(kind, v):
        k = step_no.get((kind, v), 0)
        src, r = d_in[k % n_chunks].data_ptr(), k % ring
        if kind == 'single':
            eng.session_push_device(sessions[v], src, n, d_out[r, 0].data_ptr(), cap, d_n[r, 0].data_ptr())
        else:
            eng.group_push_device(groups[v], [src] * MEMBERS, n, [d_out[r, j].data_ptr() for j in range(MEMBERS)], cap,
                                  [d_n[r, j].data_ptr() for j in range(MEMBERS)])
        step_no[(kind, v)] = k + 1

    def leg_throughput(kind, v, steps):
        eng.synchronize()
        t0 = time.perf_counter()
        done = 0
        while done < steps:
            for _ in range(min(args.block, steps - done)):
                push_device(kind, v)
            done += min(args.block, steps - done)
            eng.synchronize()
        return steps / (time.perf_counter() - t0)

    legs = [(kind, v) for kind in ('single', 'group') for v in VARIANTS]
    for leg in legs:
        leg_throughput(*leg, args.warmup)
    res = {leg: [] for leg in legs}
    for _ in range(args.repeats):
        for leg in legs:
            res[leg].append(leg_throughput(*leg, args.steps))
    meters = {v: eng.session_pitch_stats(sessions[v]) for v in VARIANTS if v != 'off'}

    # kernel time: one profiler window over the session with the correction
    from torch.profiler import ProfilerActivity, profile
    profiled = [v for v in VARIANTS if v != 'off']
    eng.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for v in profiled:
            for _ in range(args.profile_steps):
                push_device('single', v)
            eng.synchronize()
    trace = tmp / 'trace.json'
    prof.export_chrome_trace(str(trace))
    ev = json.loads(trace.read_text())
    ev = ev['traceEvents'] if isinstance(ev, dict) else ev
    kern = sorted((e for e in ev if e.get('cat') == 'kernel' and e.get('ph') == 'X'), key=lambda e: e['ts'])
    pitch_us = [e['dur'] for e in kern if KERNEL in e['name']]
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
                legs={f'{kind}_{v}': dict(steps_per_s=statistics.median(res[(kind, v)]), steps_per_s_all=res[(kind, v)])
                      for kind, v in legs},
                last_step_meter={v: dict(voiced=m[0], mean_cents=m[1], max_cents=m[2]) for v, m in meters.items()}, kernels=kernels)
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_pitch.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
