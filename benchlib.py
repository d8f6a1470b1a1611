"""What the bench_*.py scripts share: the card they ran on, the headline session, synthetic voices, device-resident steps on an output
ring, host-clock legs alternated over rounds, one profiler window's kernel durations, and the command line and its output.  torch and
the engine are imported inside the functions that use them, so a script's --help needs neither."""
import argparse
import collections
import json
import subprocess
import time
from pathlib import Path

import numpy as np

EXTRA, FS, T = (0.0, 0.5, 0.0), 24000, 0.3      # the headline stream: encode / convert / decode extras, sample rate, chunk seconds
RING = 8                                        # output slots: consecutive device-resident steps are in flight together


def card(query='name,power.limit,clocks.max.sm'):
    """The nvidia-smi fields `query` of the first card: a number is recorded with the card, power limit and clock it was measured at."""
    q = subprocess.run(['nvidia-smi', f'--query-gpu={query}', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown (nvidia-smi unavailable)'


def bench_parser(required_out=False, **defaults):
    """--out DIR, then one integer flag per keyword in the order given, each with its default."""
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, required=required_out)
    for name, default in defaults.items():
        ap.add_argument(f'--{name}', type=int, default=default)
    return ap


def require_cuda(script):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit(f'{script} needs a CUDA device')


def emit(out, name, line):
    """Write line to out / name.json when out is given, and print it as one JSON line."""
    if out is not None:
        out.mkdir(parents=True, exist_ok=True)
        (out / f'{name}.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


def headline_config(**overrides):
    """The headline session (24 kHz, 5 ms frames, 0.3 s chunks, extras 0 / 0.5 / 0, 1024-sample vocoder blocks), fields overridden."""
    from realtime_yukarin_b200.engine import SessionConfig
    cfg = dict(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
               encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
               vocoder_buffer_size=1024)
    return SessionConfig(**dict(cfg, **overrides))


def synthetic_voice(eng, tmp, seed=0):
    """A new voice of eng holding the full-width synthetic models of `seed`, written under tmp / v<seed>."""
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.models import load_voice
    paths = synthetic.write_synthetic_models(tmp / f'v{seed}', seed=seed)
    voice = eng.voice_create()
    load_voice(eng, voice, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path', 'target_statistics_path')})
    return voice


def synthetic_builtin(eng, tmp):
    """Load the full-width synthetic models of seed 0, written under tmp, as eng's built-in voice."""
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json
    paths = synthetic.write_synthetic_models(tmp, seed=0)
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=eng)
    SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=eng)


def device_chunks(x, n, count):
    """The first `count` chunks of n samples of x as one (count, n) CUDA tensor."""
    import torch
    return torch.from_numpy(np.stack([x[k * n:(k + 1) * n] for k in range(count)])).cuda()


def output_ring(cap, members=1):
    """RING output slots of `members` x `cap` samples and their sample counts, on the device."""
    import torch
    return (torch.empty((RING, members, cap), dtype=torch.float64, device='cuda'),
            torch.zeros((RING, members, 1), dtype=torch.int32, device='cuda'))


def device_pusher(eng, d_in, cap, members=1):
    """push(sid) queues the next device-resident step of a session, push(gid, group=True) that of a group whose `members` members all
    take the same chunk.  Each target counts its own steps: its step k reads chunk k mod len(d_in) and writes output slot k mod RING."""
    import torch
    n = d_in.shape[1]
    d_out, d_n = output_ring(cap, members)
    torch.cuda.synchronize()
    step_no = collections.Counter()

    def push(target, group=False):
        k = step_no[target, group]
        src, r = d_in[k % len(d_in)].data_ptr(), k % RING
        if group:
            eng.group_push_device(target, [src] * members, n, [d_out[r, j].data_ptr() for j in range(members)], cap,
                                  [d_n[r, j].data_ptr() for j in range(members)])
        else:
            eng.session_push_device(target, src, n, d_out[r, 0].data_ptr(), cap, d_n[r, 0].data_ptr())
        step_no[target, group] = k + 1
    return push


def throughput(eng, step, steps, block, launches=False):
    """steps/s of `steps` calls of step() queued in blocks of `block`, the device drained after each block as in bench.py's sustained
    figure, on the host clock from an idle device to an idle device.  With launches, (steps/s, kernels per step): the kernels are
    engine.launch_count's, read outside the timed interval because reading it synchronises the device."""
    eng.synchronize()
    launches0 = eng.launch_count if launches else None
    t0 = time.perf_counter()
    done = 0
    while done < steps:
        for _ in range(min(block, steps - done)):
            step()
        done += min(block, steps - done)
        eng.synchronize()
    rate = steps / (time.perf_counter() - t0)
    return (rate, (eng.launch_count - launches0) / steps) if launches else rate


def alternate(legs, run, steps, warmup, repeats):
    """{leg: [run(leg, steps) of each round]}: run(leg, warmup) for every leg first, then `repeats` rounds that run every leg in
    order, so that clock and neighbour drift spreads over all of them."""
    for leg in legs:
        run(leg, warmup)
    res = {leg: [] for leg in legs}
    for _ in range(repeats):
        for leg in legs:
            res[leg].append(run(leg, steps))
    return res


def stopwatch_ms(eng, step, warmup, steps):
    """`warmup` calls of step() and a device synchronise, then the device ms of `steps` more on the engine's CUDA-event stopwatch."""
    for _ in range(warmup):
        step()
    eng.synchronize()
    eng.timer_start()
    for _ in range(steps):
        step()
    return eng.timer_stop()


def kernel_events(prof, path):
    """The CUDA kernel events of a finished torch.profiler window, read back from the chrome trace it writes to path."""
    prof.export_chrome_trace(str(path))
    ev = json.loads(Path(path).read_text())
    ev = ev['traceEvents'] if isinstance(ev, dict) else ev
    return [e for e in ev if e.get('cat') == 'kernel' and e.get('ph') == 'X']


def kernel_durations(eng, tmp, run, names):
    """{name: [us of every kernel whose name contains it, in start order]} over run(), in one torch.profiler window of CUDA activity
    from an idle device to an idle device."""
    from torch.profiler import ProfilerActivity, profile
    eng.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        eng.synchronize()
    kern = sorted(kernel_events(prof, tmp / 'trace.json'), key=lambda e: e['ts'])
    return {name: [e['dur'] for e in kern if name in e['name']] for name in names}
