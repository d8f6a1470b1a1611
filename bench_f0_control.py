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
import argparse
import json
import shutil
import statistics
import subprocess
import tempfile
import time
from pathlib import Path

import numpy as np

EXTRA, FS, T = (0.0, 0.5, 0.0), 24000, 0.3
VARIANTS = ('off', 'measure', 'follow', 'set')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown (nvidia-smi unavailable)'


def make_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, default=None)
    ap.add_argument('--steps', type=int, default=3000)
    ap.add_argument('--block', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=40)
    ap.add_argument('--repeats', type=int, default=3)
    return ap


def main(argv=None):
    args = make_parser().parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_f0_control.py needs a CUDA device')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import load_voice

    tmp = Path(tempfile.mkdtemp(prefix='bench_f0_control_'))        # synthetic model files: never written into the tree
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
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    d_in = torch.from_numpy(np.stack([x[k * n:(k + 1) * n] for k in range(n_chunks)])).cuda()
    sids = {}
    for v in VARIANTS:
        sids[v] = eng.session_create(cfg, voice=voice)
        if v in ('measure', 'follow'):
            eng.session_f0_measure(sids[v])
        if v == 'follow':
            eng.session_f0_follow(sids[v], True, min_voiced_frames=200)
    cap = eng.session_io_geometry(sids['off'])['max_out']
    ring = 8                                      # distinct output slots: consecutive steps are in flight together
    d_out = torch.empty((ring, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((ring, 1), dtype=torch.int32, device='cuda')
    step_no = {v: 0 for v in VARIANTS}
    base_map = eng.session_get_f0_map(sids['set'])

    def push(v):
        k = step_no[v]
        if v == 'set':                            # a different map every step, so that every step stages a copy
            eng.session_set_f0_map(sids[v], target_mean=base_map['target_mean'], semitones=(k % 5) - 2)
        eng.session_push_device(sids[v], d_in[k % n_chunks].data_ptr(), n, d_out[k % ring].data_ptr(), cap, d_n[k % ring].data_ptr())
        step_no[v] = k + 1

    def leg(v, steps):
        eng.synchronize()
        launches0 = eng.launch_count
        t0 = time.perf_counter()
        done = 0
        while done < steps:
            for _ in range(min(args.block, steps - done)):
                push(v)
            done += min(args.block, steps - done)
            eng.synchronize()
        s = time.perf_counter() - t0
        return steps / s, (eng.launch_count - launches0) / steps

    for v in VARIANTS:
        leg(v, args.warmup)
    rates = {v: [] for v in VARIANTS}
    kernels = {}
    for _ in range(args.repeats):
        for v in VARIANTS:
            r, kernels[v] = leg(v, args.steps)
            rates[v].append(r)
    measured = {v: eng.session_f0_measured(sids[v]) for v in ('measure', 'follow')}
    for sid in sids.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, block=args.block, warmup=args.warmup, repeats=args.repeats,
                variants={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=kernels[v])
                          for v in VARIANTS},
                voiced_frames_counted={v: m[0] for v, m in measured.items()})
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_f0_control.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
