"""Cost of the output limiter on the headline stream (precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic
voice): steps/s of device-resident ryk_session_push_device steps in blocks of --block (the device drains between blocks, as in bench.py's
sustained figure) for sessions returning 24 kHz and 48 kHz, each without the limiter and with it at a 5 ms look-ahead and a hold of 50
and of 500 ms.  The limiter runs at a gain under which the voice plays 4x over the -1 dB ceiling, so it limits on every step.

The variants alternate within each of --repeats rounds after --warmup steps each.  After the timed rounds one torch.profiler window over
--profile_steps steps of each limited session gives the three limiter kernels' device time per step, next to the synthesis stage's
other kernels.  The card's name and power limit are recorded with the numbers.

    python bench_limiter.py [--out DIR] [--steps 1000 --block 100 --warmup 30 --repeats 3 --profile_steps 20]

Prints one JSON line (and writes it to DIR/bench_limiter.json with --out).  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from bench_f0_control import EXTRA, FS, T, card

VARIANTS = [(rate, hold) for rate in (24000, 48000) for hold in (None, 50.0, 500.0)]
LOOKAHEAD_MS = 5.0
KERNELS = ('k_lim_g0', 'k_lim_min', 'k_lim_apply')


def _name(v):
    rate, hold = v
    return f'{rate // 1000}k_' + ('off' if hold is None else f'hold{int(hold)}')


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
        raise SystemExit('bench_limiter.py needs a CUDA device')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import load_voice

    tmp = Path(tempfile.mkdtemp(prefix='bench_limiter_'))           # synthetic model files: never written into the tree
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
    cap = max(eng.session_io_geometry(s)['max_out'] for s in sessions.values())
    ring = 8                                      # distinct output slots: consecutive steps are in flight together
    d_out = torch.empty((ring, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((ring, 1), dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    step_no = {v: 0 for v in VARIANTS}

    def push_device(v):
        k = step_no[v]
        eng.session_push_device(sessions[v], d_in[k % n_chunks].data_ptr(), n, d_out[k % ring].data_ptr(), cap, d_n[k % ring].data_ptr())
        step_no[v] = k + 1

    def leg_throughput(v, steps):
        eng.synchronize()
        t0 = time.perf_counter()
        done = 0
        while done < steps:
            for _ in range(min(args.block, steps - done)):
                push_device(v)
            done += min(args.block, steps - done)
            eng.synchronize()
        return steps / (time.perf_counter() - t0)

    for v in VARIANTS:
        leg_throughput(v, args.warmup)
    res = {v: [] for v in VARIANTS}
    for _ in range(args.repeats):
        for v in VARIANTS:
            res[v].append(leg_throughput(v, args.steps))
    reductions = {_name(v): eng.session_limiter_stats(sessions[v]) for v in VARIANTS if v[1] is not None}

    # kernel times: one profiler window, one limited session after the other
    from torch.profiler import ProfilerActivity, profile
    limited = [v for v in VARIANTS if v[1] is not None]
    eng.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for v in limited:
            for _ in range(args.profile_steps):
                push_device(v)
            eng.synchronize()
    trace = tmp / 'trace.json'
    prof.export_chrome_trace(str(trace))
    ev = json.loads(trace.read_text())
    ev = ev['traceEvents'] if isinstance(ev, dict) else ev
    kern = sorted((e for e in ev if e.get('cat') == 'kernel' and e.get('ph') == 'X'), key=lambda e: e['ts'])
    kernels = {}
    for i, v in enumerate(limited):
        per = {}
        for name in KERNELS:
            d = [e['dur'] for e in kern if name in e['name']][i * args.profile_steps:(i + 1) * args.profile_steps]
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
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_limiter.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
